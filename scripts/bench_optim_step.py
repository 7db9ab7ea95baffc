#!/usr/bin/env python
"""The optimiser step of a fused-engine training step: torch.optim (the engine re-packs itself through refresh() on the next
forward, and packs its W^T operands again in the first backward) against openscene_b200.optim bound to the engine (one
update launch, one in-place re-pack launch).

    python scripts/bench_optim_step.py [--steps K] [--warmup W] [--out DIR]

Workloads: ``distill.fused_distill_step`` with Adam(lr 1e-3) for MinkUNet18A and MinkUNet34C on synth.scene('config2_200k'),
feats = 1, 20,000 supervised rows, 768-d targets (the scene of scripts/bench_train_step.py); ``train_mink.fused_train_step``
with SGD(lr 0.01, momentum 0.9, weight decay 1e-4) for MinkUNet18A with 20 classes on 8 config1_50k scenes (the batch of
scripts/bench_train_mink_step.py).  Each arm owns a copy of the model, its engine and its optimiser; before every step the
weights, buffers and optimiser state are restored in place from the same snapshot and the L2 is flushed (256 MiB memset),
outside the step's CUDA-event pair, and the arms alternate.  The bound arm's engine is brought up to the restored weights by
its own in-place re-pack outside the event pair; the torch arm's engine re-packs inside the step, as it does after every
torch.optim step in training.

Reported per workload and arm: ms per step (min / median / max); the optimiser plus re-pack alone ('opt_ms': torch's
step() + refresh() + the lazy W^T packs, against the bound step()), CUDA events around that work only, median of 10 with the
gradients of a real backward in place; libosb200 launches per training step (osb_launch_count); peak memory per step; the
device name, power limit and SM clock of the same run.  The JSON line is printed and, with --out, written to
DIR/bench_optim_step.json."""
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


def _median(pairs):
    ts = sorted(a.elapsed_time(b) for a, b in pairs)
    return {'ms_min': ts[0], 'ms_median': ts[len(ts) // 2], 'ms_max': ts[-1]}


class Arm:
    def __init__(self, base, bound, make_opt, step_fn, dev):
        from openscene_b200 import engine
        self.model = copy.deepcopy(base).to(dev)
        self.eng = engine.FusedMinkUNet(self.model, batch_stats=True)
        self.opt = make_opt(self.model.parameters())
        self.bound = bound
        if bound:
            self.opt.bind(self.eng)
        self.fn = lambda: step_fn(self.eng, self.opt)
        self.fn()                                          # optimiser state and W^T packs exist
        torch.cuda.synchronize()
        self.snap_m = {k: v.clone() for k, v in self.model.state_dict().items()}
        self.snap_o = {id(p): {k: (v.clone() if torch.is_tensor(v) else v) for k, v in self.opt.state[p].items()}
                       for p in self.model.parameters()}

    def restore(self):
        with torch.no_grad():
            for k, v in self.model.state_dict().items():
                v.copy_(self.snap_m[k])
            for p in self.model.parameters():
                for k, v in self.opt.state[p].items():
                    if torch.is_tensor(v):
                        v.copy_(self.snap_o[id(p)][k])
        if self.bound:
            self.opt.repack_bound()                        # the engine follows the restored weights in place

    def opt_alone(self):
        """CUDA-event time of the optimiser and everything it makes the engine redo, with real gradients in place"""
        from openscene_b200 import engine_train
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if self.bound:
            a.record(); self.opt.step(); b.record()
            return a, b
        widths = [[hi - lo for (lo, hi, _) in cv.bwd] if isinstance(cv.bwd, list) else None for cv in self.eng._bwd_convs]
        a.record()
        self.opt.step()
        self.eng.refresh()
        engine_train._ensure_bwd_packs(self.eng)
        for cv, w in zip(self.eng._bwd_convs, widths):
            if w is not None:
                engine_train._packs_for(cv, w)
        b.record()
        return a, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from bench_batch_stats import power_limit_w
    from bench_train_mink_step import labels_for
    from openscene_b200 import _cabi as C
    from openscene_b200 import distill, optim, synth, train_mink
    assert torch.cuda.is_available(), "bench_optim_step.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)

    coords = torch.from_numpy(synth.scene('config2_200k', seed=0)).to(dev)
    feats = torch.ones(coords.shape[0], 3, device=dev)
    g = torch.Generator().manual_seed(0)
    mask = torch.zeros(coords.shape[0], dtype=torch.bool)
    mask[torch.randperm(coords.shape[0], generator=g)[:20000]] = True
    mask = mask.to(dev)
    tgt = torch.randn(20000, 768, generator=g).half().to(dev)
    ce_c = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=s, batch_index=s)) for s in range(8)])
    ce_f = torch.rand(len(ce_c), 3, generator=torch.Generator().manual_seed(2)).to(dev)
    ce_l = labels_for(ce_c, 20).to(dev)
    ce_c = ce_c.to(dev)

    distill_fn = lambda eng, opt: distill.fused_distill_step(eng, opt, coords, feats, tgt, mask, translate=False)
    ce_fn = lambda eng, opt: train_mink.fused_train_step(eng, opt, ce_c, ce_f, ce_l, translate=False)
    sgd_kw = dict(lr=0.01, momentum=0.9, weight_decay=1e-4)
    workloads = {
        'distill_MinkUNet18A_adam': ('MinkUNet18A', 768, distill_fn, lambda ps: torch.optim.Adam(ps, lr=1e-3),
                                     lambda ps: optim.Adam(ps, lr=1e-3)),
        'distill_MinkUNet34C_adam': ('MinkUNet34C', 768, distill_fn, lambda ps: torch.optim.Adam(ps, lr=1e-3),
                                     lambda ps: optim.Adam(ps, lr=1e-3)),
        'train_mink_MinkUNet18A_sgd': ('MinkUNet18A', 20, ce_fn, lambda ps: torch.optim.SGD(ps, **sgd_kw),
                                       lambda ps: optim.SGD(ps, **sgd_kw)),
    }
    result = {'metric': 'ms per training step, torch.optim (engine re-packs via refresh) vs openscene_b200.optim bound',
              'distill_scene': f'config2_200k, {coords.shape[0]} voxels, feats = 1, 20000 supervised rows, 768-d targets',
              'train_mink_batch': f'8 x config1_50k, {ce_c.shape[0]} voxels, 20 classes, 10 % ignore label 255',
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w, 'power_limit_source': power_how,
              'steps': args.steps, 'warmup': args.warmup,
              'method': 'weights, buffers and optimiser state restored in place and L2 flushed before every step, outside '
                        'the CUDA-event pair; arms alternate', 'workloads': {}}

    for name, (arch, out, fn, torch_opt, our_opt) in workloads.items():
        base = synth.build_model(arch, out, seed=0).train()
        arms = {'torch_optim': Arm(base, False, torch_opt, fn, dev), 'bound': Arm(base, True, our_opt, fn, dev)}
        for _ in range(args.warmup):
            for arm in arms.values():
                arm.restore()
                arm.fn()
        rec = {}
        # one step from the same state: losses and parameters of the two arms
        losses = {}
        for k, arm in arms.items():
            arm.restore()
            r = arm.fn()
            losses[k] = float(r[0] if isinstance(r, tuple) else r)
        pa, pb = list(arms['torch_optim'].model.parameters()), list(arms['bound'].model.parameters())
        rec['loss'] = losses
        rec['params_bit_equal_fraction'] = sum(int((a == b).sum()) for a, b in zip(pa, pb)) / sum(a.numel() for a in pa)
        # launches per step
        launches = {}
        for k, arm in arms.items():
            arm.restore()
            torch.cuda.synchronize()
            n0 = C.lib().osb_launch_count()
            arm.fn()
            launches[k] = C.lib().osb_launch_count() - n0
        rec['osb_launches_per_step'] = launches
        # the optimiser and the re-pack alone, gradients of a real backward in place
        alone = {k: [] for k in arms}
        for _ in range(10):
            for k, arm in arms.items():
                arm.restore()
                arm.fn()
                flush.zero_()
                alone[k].append(arm.opt_alone())
        torch.cuda.synchronize()
        rec['opt_ms'] = {k: _median(v) for k, v in alone.items()}
        evs, peak = {k: [] for k in arms}, {}
        gc.collect()
        gc.disable()
        try:
            for i in range(args.steps):
                for k, arm in arms.items():
                    arm.restore()
                    flush.zero_()
                    torch.cuda.reset_peak_memory_stats(dev)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); arm.fn(); b.record()
                    evs[k].append((a, b))
                    if i == 0:
                        torch.cuda.synchronize()
                        peak[k] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
                if i in (args.steps // 4, args.steps // 2, (3 * args.steps) // 4):
                    sampler.sample()
            torch.cuda.synchronize()
        finally:
            gc.enable()
        for k in arms:
            rec[k] = _median(evs[k])
        rec['peak_mem_gib'] = peak
        rec['step_saving_ms_median'] = rec['torch_optim']['ms_median'] - rec['bound']['ms_median']
        result['workloads'][name] = rec
        print(name, json.dumps(rec), flush=True)
        del arms, base
        torch.cuda.empty_cache()
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_optim_step.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
