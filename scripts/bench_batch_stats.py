#!/usr/bin/env python
"""Train-mode forward under no_grad (run/distill.py's validate(): BatchNorm with batch statistics, running buffers moved) on
the bench scene: the module-by-module path against ``FusedMinkUNet(model, batch_stats=True)``.

    python scripts/bench_batch_stats.py [--steps K] [--warmup W] [--out DIR]

Scene: synth.scene('config2_200k') (the bench.py workload), feats = 1, MinkUNet18A (the ScanNet distill architecture) and
MinkUNet34C, 768-d head.  Before every step the running buffers are restored from a snapshot (both arms see the same state)
and the L2 is flushed (256 MiB memset), both outside the step's CUDA-event pair; the arms alternate step by step.  For scale,
a third arm times the eval-mode engine on the same per-layer launch path (persistent chain off): the difference to the
batch-statistics arm is what the reductions and apply passes cost.

Reported per architecture: ms per scene (min / median / max) of each arm, the max per-row relative difference between the
two train-mode outputs, launches per step; and the device name, power limit and SM clock.  The power limit is read before
the timed region, the SM clock on the device between steps (bench.py's ClockSampler), so no query overlaps a timed step.
The JSON line is printed and, with --out, written to DIR/bench_batch_stats.json."""
import argparse
import copy
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def power_limit_w(index):
    """(power limit in W, how it was read); None when neither NVML nor nvidia-smi answers"""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        return pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0, 'nvml'
    except Exception:                                        # noqa: BLE001
        pass
    try:
        r = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=60)
        return float(r.stdout.strip().splitlines()[0]), 'nvidia-smi'
    except Exception:                                        # noqa: BLE001
        return None, 'unavailable'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--archs', default='MinkUNet18A,MinkUNet34C')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import MinkowskiEngine as ME
    from bench import ClockSampler
    from openscene_b200 import _cabi, engine, synth
    assert torch.cuda.is_available(), "bench_batch_stats.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    coords = torch.from_numpy(synth.scene('config2_200k', seed=0)).to(dev)
    feats = torch.ones(coords.shape[0], 3, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)
    result = {'metric': 'ms per scene, train-mode forward under no_grad (batch-statistics BatchNorm)',
              'scene': f'config2_200k, {coords.shape[0]} voxels, feats = 1, 768-d head',
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w, 'power_limit_source': power_how,
              'steps': args.steps, 'warmup': args.warmup,
              'method': 'running buffers restored and L2 flushed before every step, outside the CUDA-event pair; arms alternate',
              'archs': {}}

    for arch in args.archs.split(','):
        model = synth.build_model(arch, 768, seed=0).train().to(dev)
        bufs = [b for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)
                for b in (m.running_mean, m.running_var, m.num_batches_tracked)]
        snap = [b.clone() for b in bufs]
        eng = engine.FusedMinkUNet(model, batch_stats=True)
        ev_model = copy.deepcopy(model).eval()
        eng_eval = engine.FusedMinkUNet(ev_model)
        eng_eval.use_chain = False                            # the per-layer launch path the batch-statistics mode uses

        def restore():
            with torch.no_grad():
                for b, s in zip(bufs, snap):
                    b.copy_(s)

        def module_arm():
            with torch.no_grad():
                return model(ME.SparseTensor(feats, coords))

        arms = {'module_path': module_arm, 'engine_batch_stats': lambda: eng(coords, feats),
                'eval_engine_per_layer': lambda: eng_eval(coords, feats)}
        for _ in range(args.warmup):
            for fn in arms.values():
                restore()
                fn()
        torch.cuda.synchronize()
        restore()
        ref = module_arm()
        restore()
        out = eng(coords, feats)
        err = float(((out.double() - ref.double()).norm(dim=1) / (ref.double().norm(dim=1) + 1e-30)).max())
        torch.cuda.synchronize()

        launches = {}
        for name, fn in arms.items():
            l0 = _cabi.lib().osb_launch_count()
            fn()
            torch.cuda.synchronize()
            launches[name] = int(_cabi.lib().osb_launch_count() - l0)
        evs = {name: [] for name in arms}
        gc.collect()
        gc.disable()
        try:
            for i in range(args.steps):
                for name, fn in arms.items():
                    restore()
                    flush.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); fn(); b.record()
                    evs[name].append((a, b))
                if i in (args.steps // 4, args.steps // 2, (3 * args.steps) // 4):
                    sampler.sample()                          # stream-ordered between steps, outside every event pair
            torch.cuda.synchronize()
        finally:
            gc.enable()
        rec = {'rel_row_err_engine_vs_module': err, 'launches_per_step': launches}
        for name, pairs in evs.items():
            ts = sorted(a.elapsed_time(b) for a, b in pairs)
            rec[name] = {'ms_min': ts[0], 'ms_median': ts[len(ts) // 2], 'ms_max': ts[-1]}
        rec['speedup_median'] = rec['module_path']['ms_median'] / rec['engine_batch_stats']['ms_median']
        result['archs'][arch] = rec
        restore()
        del eng, eng_eval, ev_model, model
        torch.cuda.empty_cache()
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_batch_stats.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
