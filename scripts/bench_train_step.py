#!/usr/bin/env python
"""One distillation training step (run/distill.py: translate, forward, cosine loss on the supervised rows, backward, Adam) on
the bench scene: ``distill.distill_step`` on the module path against ``distill.fused_distill_step`` on
``FusedMinkUNet(model, batch_stats=True)``.

    python scripts/bench_train_step.py [--steps K] [--warmup W] [--out DIR]

Scene: synth.scene('config2_200k'), feats = 1, 20,000 supervised rows, 768-d targets, MinkUNet18A and MinkUNet34C.  Each arm
owns a copy of the model and of its Adam state; before every step both are restored from the same snapshot and the L2 is
flushed (256 MiB memset), outside the step's CUDA-event pair, and the arms alternate.  Restoring the weights makes the engine
re-pack inside the step, as an optimiser step does in training; the re-pack of the forward operands is also timed alone
('repack_ms'; the W^T operands of the dgrads are packed inside the first backward after it and are not part of that number).

Reported per architecture: ms per step (min / median / max) of each arm, the re-pack time and its share of the engine step, peak
memory per step, the loss difference and the largest per-parameter gradient difference (relative to that parameter's largest
gradient) after one step from the same state; and the device name, power limit and SM clock.  The JSON line is printed and,
with --out, written to DIR/bench_train_step.json."""
import argparse
import copy
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--archs', default='MinkUNet18A,MinkUNet34C')
    ap.add_argument('--rows', type=int, default=20000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from bench_batch_stats import power_limit_w
    from openscene_b200 import distill, engine, engine_train, synth
    assert torch.cuda.is_available(), "bench_train_step.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    coords = torch.from_numpy(synth.scene('config2_200k', seed=0)).to(dev)
    feats = torch.ones(coords.shape[0], 3, device=dev)
    g = torch.Generator().manual_seed(0)
    mask = torch.zeros(coords.shape[0], dtype=torch.bool)
    mask[torch.randperm(coords.shape[0], generator=g)[:args.rows]] = True
    mask = mask.to(dev)
    tgt = torch.randn(args.rows, 768, generator=g).half().to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)
    result = {'metric': 'ms per training step (translate, forward, cosine loss, backward, Adam)',
              'scene': f'config2_200k, {coords.shape[0]} voxels, feats = 1, {args.rows} supervised rows, 768-d targets',
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w, 'power_limit_source': power_how,
              'steps': args.steps, 'warmup': args.warmup,
              'method': 'weights, buffers and Adam state restored and L2 flushed before every step, outside the CUDA-event '
                        'pair; arms alternate',
              'archs': {}}

    for arch in args.archs.split(','):
        base = synth.build_model(arch, 768, seed=0).train().to(dev)
        m_mod, m_eng = copy.deepcopy(base), copy.deepcopy(base)
        o_mod, o_eng = torch.optim.Adam(m_mod.parameters(), lr=1e-3), torch.optim.Adam(m_eng.parameters(), lr=1e-3)
        eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
        distill.distill_step(m_mod, o_mod, coords, feats, tgt, mask)             # Adam state exists in both arms
        distill.fused_distill_step(eng, o_eng, coords, feats, tgt, mask)
        snap_m = copy.deepcopy(base.state_dict())
        snap_o = copy.deepcopy(o_mod.state_dict())

        def restore(m, o):
            with torch.no_grad():
                for k, v in m.state_dict().items():
                    v.copy_(snap_m[k])
            o.load_state_dict(snap_o)

        arms = {'module_path': (m_mod, o_mod, lambda: distill.distill_step(m_mod, o_mod, coords, feats, tgt, mask)),
                'engine': (m_eng, o_eng, lambda: distill.fused_distill_step(eng, o_eng, coords, feats, tgt, mask))}
        for _ in range(args.warmup):
            for m, o, fn in arms.values():
                restore(m, o)
                fn()
        # one step from the same state without the update: loss and gradient differences
        losses, grads = {}, {}
        for name, (m, o, _) in arms.items():
            restore(m, o)
            keep = torch.optim.SGD(m.parameters(), lr=0.0)
            keep.step = lambda closure=None: None
            torch.manual_seed(1)
            losses[name] = float(distill.distill_step(m, keep, coords, feats, tgt, mask) if name == 'module_path'
                                 else distill.fused_distill_step(eng, keep, coords, feats, tgt, mask))
            grads[name] = [p.grad.clone() for p in m.parameters()]
        gdiff = max(float((a - b).abs().max() / (b.abs().max() + 1e-30)) for a, b in zip(grads['engine'], grads['module_path']))
        del grads
        # re-pack alone
        rp = []
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); eng.refresh(); engine_train._ensure_bwd_packs(eng); b.record()
            rp.append((a, b))
        torch.cuda.synchronize()
        repack = sorted(a.elapsed_time(b) for a, b in rp)[2]
        evs, peak = {n: [] for n in arms}, {}
        gc.collect()
        gc.disable()
        try:
            for i in range(args.steps):
                for name, (m, o, fn) in arms.items():
                    restore(m, o)
                    flush.zero_()
                    torch.cuda.reset_peak_memory_stats(dev)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); fn(); b.record()
                    evs[name].append((a, b))
                    if i == 0:
                        torch.cuda.synchronize()
                        peak[name] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
                if i in (args.steps // 4, args.steps // 2, (3 * args.steps) // 4):
                    sampler.sample()
            torch.cuda.synchronize()
        finally:
            gc.enable()
        rec = {'loss_module': losses['module_path'], 'loss_engine': losses['engine'],
               'loss_rel_diff': abs(losses['engine'] - losses['module_path']) / abs(losses['module_path']),
               'max_param_grad_diff_rel_to_max': gdiff, 'repack_ms': repack, 'peak_mem_gib': peak}
        for name, pairs in evs.items():
            ts = sorted(a.elapsed_time(b) for a, b in pairs)
            rec[name] = {'ms_min': ts[0], 'ms_median': ts[len(ts) // 2], 'ms_max': ts[-1]}
        rec['repack_share_of_engine_step'] = repack / rec['engine']['ms_median']
        rec['speedup_median'] = rec['module_path']['ms_median'] / rec['engine']['ms_median']
        result['archs'][arch] = rec
        del eng, m_mod, m_eng, o_mod, o_eng, base
        torch.cuda.empty_cache()
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_train_step.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
