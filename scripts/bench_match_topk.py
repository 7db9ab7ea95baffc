#!/usr/bin/env python
"""Open-vocabulary matching for large label sets: ``matching.match_topk`` (osb_match_topk, the [N_pts, K] scores never in
memory) against torch in 4,096-row text chunks (``X[inds_reverse].half() @ T_chunk.t()``, ``topk``, merge of the chunk
results) and, where it fits, torch's full product ``(X[inds_reverse].half() @ T.t()).topk(k)`` as run/evaluate.py takes it.

    python scripts/bench_match_topk.py [--reps R] [--rounds N] [--out DIR]

Points: the raw points of synth.scene_points('config2_200k') voxelised at its 2 cm voxel, fp32 features [n_vox, 768] gathered
through inds_reverse.  Sizes: K in {20, 160, 1203, 20000}, k in {1, 5}.  The arms alternate per round; each round times R
back-to-back calls between two CUDA events.  Peak memory per arm is ``max_memory_allocated`` above the inputs in a separate
call.  The full product is skipped where its [N_pts, K] fp16 scores would exceed --full-gib.

Also reported: the operation count 2 N_pts K C, the L2 -> SM text traffic (each 128-point CTA streams all of T:
ceil(N_pts / 128) * K * C * 2 bytes) and the HBM bytes (the gathered features once, T once), each over the median time, with
the device name, power limit and SM clocks sampled during the run.  The JSON line is printed and, with --out, written to
DIR/bench_match_topk.json."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

CHUNK = 4096


def torch_chunked(x, inv, text, k):
    a = x[inv].half()
    best_v, best_i = None, None
    for j in range(0, text.shape[0], CHUNK):
        v, i = (a @ text[j:j + CHUNK].t()).topk(min(k, text[j:j + CHUNK].shape[0]), dim=1)
        i = i + j
        if best_v is None:
            best_v, best_i = v, i
        else:
            v, sel = torch.cat([best_v, v], 1).topk(k, dim=1)
            best_v, best_i = v, torch.cat([best_i, i], 1).gather(1, sel)
    return best_v, best_i


def torch_full(x, inv, text, k):
    return (x[inv].half() @ text.t()).topk(k, dim=1)


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    del out
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ks', type=int, nargs='+', default=[20, 160, 1203, 20000])
    ap.add_argument('--topk', type=int, nargs='+', default=[1, 5])
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--full-gib', type=float, default=8.0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from bench_batch_stats import power_limit_w
    from openscene_b200 import matching, synth
    assert torch.cuda.is_available(), "bench_match_topk.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    pts, voxel = synth.scene_points('config2_200k')
    _, inv = np.unique(np.floor(pts / voxel).astype(np.int64), axis=0, return_inverse=True)
    inv = torch.from_numpy(inv.reshape(-1)).to(dev)
    n_pts, n_vox, c = inv.shape[0], int(inv.max()) + 1, 768
    x = torch.randn(n_vox, c, generator=torch.Generator().manual_seed(0)).to(dev)
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)
    result = {'metric': 'per-point top-k of the open-vocabulary match: device streaming top-k vs torch',
              'workload': f'synth config2_200k: {n_pts} points, {n_vox} voxels, C = {c}, fp32 features via inds_reverse',
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w, 'power_limit_source': power_how,
              'reps_per_round': args.reps, 'rounds': args.rounds, 'runs': {}}
    for K in args.ks:
        text = torch.from_numpy(synth.text_embeddings(K, c)).to(dev)
        for k in args.topk:
            arms = {'match_topk': lambda: matching.match_topk(x, inv, text, k=k),
                    'torch_chunked_4096': lambda: torch_chunked(x, inv, text, k)}
            if n_pts * K * 2 / 2 ** 30 <= args.full_gib:
                arms['torch_full'] = lambda: torch_full(x, inv, text, k)
            # agreement on this workload: labels[:, 0] against the chunked torch arm (ties and rounding order aside)
            l_dev = matching.match_topk(x, inv, text, k=k)[1]
            l_ref = torch_chunked(x, inv, text, k)[1]
            agree = float((l_dev[:, 0] == l_ref[:, 0]).float().mean())
            del l_dev, l_ref
            mem = {n: peak(fn) for n, fn in arms.items()}
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            times = {n: [] for n in arms}
            for _ in range(args.rounds):
                for n, fn in arms.items():
                    times[n].append(timed(fn, args.reps))
                sampler.sample()
            med = statistics.median(times['match_topk'])
            flop = 2.0 * n_pts * K * c
            l2_bytes = float(-(-n_pts // 128)) * K * c * 2
            hbm_bytes = float(n_pts) * c * 4 + K * c * 2
            result['runs'][f'K={K},k={k}'] = {
                **{n: {'ms_min': min(t), 'ms_median': statistics.median(t), 'ms_max': max(t), 'peak_mib': mem[n]}
                   for n, t in times.items()},
                'match_topk_tflops': flop / med / 1e9, 'match_topk_l2_text_gbps': l2_bytes / med / 1e6,
                'match_topk_hbm_gbps': hbm_bytes / med / 1e6, 'label0_agreement_vs_torch': agree}
        del text
        torch.cuda.empty_cache()
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_match_topk.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
