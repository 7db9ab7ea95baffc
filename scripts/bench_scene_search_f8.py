"""FP8 scene index: ``SceneIndex(storage='fp8')`` against the fp16 index on the workloads of bench_scene_search.py and
bench_scene_regions.py, in one run.

- Search: 64 scenes of 196,000 seeded random rows (C = 768), k = 32, nq = 1 / 20 / 96.
- Regions: 64 ``synth.scene('config2_200k')`` scenes with planted boxes (as bench_scene_regions.py), threshold 0.5,
  reach 1, R = 8.
- Capacity: one FP8 index of 128 search scenes (about the memory of the 64-scene fp16 index), queried at each nq.

The fp16 and FP8 arms alternate and are timed with CUDA events (medians and ranges).  Per arm: index bytes and the achieved
rate of index read; a 1 GiB device-to-device copy in the same run is the bandwidth yardstick.  Agreement between the fp16
index on the source rows and the FP8 index (top-k overlap, top-1, scene argmax, score differences) is reported, not
asserted: the rows are seeded random rows, not OpenScene features.  Also the rate at which ``add`` quantizes rows.

    python scripts/bench_scene_search_f8.py --out DIR [--scenes 64] [--rows-per-scene 196000] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

THR, R, ANCHORS = 0.5, 8, 4


def smi(fields):
    try:
        return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f'unavailable: {e}'


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def med(v):
    return sorted(v)[len(v) // 2]


def alternate(arms, reps):
    """arms: name -> fn; warmed, then timed in turn reps times -> name -> (times, last output)"""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    t = {k: [] for k in arms}
    out = {}
    for _ in range(reps):
        for k, fn in arms.items():
            dt, out[k] = timed(fn)
            t[k].append(dt)
    return t, out


def row_bytes(storage, c, coords=False):
    return (2 * c + 4 if storage == 'fp16' else c + 5) + (16 if coords else 0)


def search_rows(s, n, c, dev):
    gen = torch.Generator(device=dev).manual_seed(s)
    return (torch.randn(n, c, generator=gen, device=dev) * 0.05).half()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--scenes', type=int, default=64)
    ap.add_argument('--rows-per-scene', type=int, default=196_000)
    ap.add_argument('--capacity-scenes', type=int, default=128)
    ap.add_argument('--channels', type=int, default=768)
    ap.add_argument('--k', type=int, default=32)
    ap.add_argument('--nq', type=int, nargs='+', default=[1, 20, 96])
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    os.makedirs(a.out, exist_ok=True)
    import __graft_entry__ as g
    g.build()
    from openscene_b200 import synth
    from openscene_b200.search import SceneIndex
    dev, C = torch.device('cuda:0'), a.channels
    res = {'info': {'device': torch.cuda.get_device_name(0),
                    'power_limit_and_max_sm_clock': smi('power.limit,clocks.max.sm')},
           'note': 'agreement figures are on seeded random rows, not OpenScene features'}
    src = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    t, _ = alternate({'copy': lambda: dst.copy_(src)}, a.reps)
    res['d2d_copy_GBps_read_plus_write'] = 2 * src.numel() / (med(t['copy']) * 1e-3) / 1e9
    del src, dst

    # ---------------- search workload
    n = a.scenes * a.rows_per_scene
    idx = {'fp16': SceneIndex(n, C, device=dev), 'fp8': SceneIndex(n, C, device=dev, storage='fp8')}
    tq = []
    for s in range(a.scenes):
        rows = search_rows(s, a.rows_per_scene, C, dev)
        idx['fp16'].add(rows)
        dt, _ = timed(lambda: idx['fp8'].add(rows))
        tq.append(dt)
    res['quantize_add_GBps_fp16_rows_in'] = n * 2 * C / (sum(tq) * 1e-3) / 1e9
    res['search'] = {'rows': n, 'scenes': a.scenes, 'k': a.k, 'runs': [],
                     'index_bytes': {k: n * row_bytes(k, C) for k in idx}}
    off = torch.tensor(idx['fp16']._off, device=dev)
    for nq in a.nq:
        q = torch.randn(nq, C, generator=torch.Generator(device=dev).manual_seed(1000 + nq), device=dev).half()
        t, out = alternate({k: (lambda i=i: i.query(q, k=a.k)) for k, i in idx.items()}, a.reps)
        r16, r8 = out['fp16'], out['fp8']
        g16, g8 = off[r16.scene.clamp(min=0)] + r16.row, off[r8.scene.clamp(min=0)] + r8.row
        overlap = [len(set(g16[j].tolist()) & set(g8[j].tolist())) / a.k for j in range(nq)]
        r = {'nq': nq, 'sm_clock_now': smi('clocks.sm')}
        for k in idx:
            r[k] = {'ms_median': med(t[k]), 'ms_range': [min(t[k]), max(t[k])],
                    'index_read_GBps': n * row_bytes(k, C) / (med(t[k]) * 1e-3) / 1e9}
        r['agreement'] = {'topk_overlap_mean': float(np.mean(overlap)), 'topk_overlap_min': float(np.min(overlap)),
                          'top1': float((g16[:, 0] == g8[:, 0]).float().mean()),
                          'scene_argmax': float((r16.scene_argmax == r8.scene_argmax).float().mean()),
                          'max_abs_topk_score_diff_by_rank': float((r16.score.float() - r8.score.float()).abs().max()),
                          'max_abs_scene_max_diff': float((r16.scene_max.float() - r8.scene_max.float()).abs().max())}
        res['search']['runs'].append(r)
        print(json.dumps(r), flush=True)
    del idx, off
    torch.cuda.empty_cache()

    # ---------------- capacity: one FP8 index of capacity-scenes search scenes
    n_cap = a.capacity_scenes * a.rows_per_scene
    big = SceneIndex(n_cap, C, device=dev, storage='fp8')
    for s in range(a.capacity_scenes):
        big.add(search_rows(s, a.rows_per_scene, C, dev))
    torch.cuda.synchronize()
    res['capacity'] = {'rows': n_cap, 'scenes': a.capacity_scenes, 'index_bytes': n_cap * row_bytes('fp8', C),
                       'allocated_bytes': torch.cuda.memory_allocated(), 'runs': []}
    for nq in a.nq:
        q = torch.randn(nq, C, generator=torch.Generator(device=dev).manual_seed(1000 + nq), device=dev).half()
        t, _ = alternate({'fp8': lambda: big.query(q, k=a.k)}, a.reps)
        r = {'nq': nq, 'ms_median': med(t['fp8']), 'ms_range': [min(t['fp8']), max(t['fp8'])],
             'index_read_GBps': n_cap * row_bytes('fp8', C) / (med(t['fp8']) * 1e-3) / 1e9}
        res['capacity']['runs'].append(r)
        print(json.dumps({'capacity': r}), flush=True)
    del big
    torch.cuda.empty_cache()

    # ---------------- regions workload (bench_scene_regions.py's data)
    cs = [synth.scene('config2_200k', seed=s)[:, 1:] for s in range(a.scenes)]
    n = sum(len(c) for c in cs)
    idx = {'fp16': SceneIndex(n, C, device=dev, coords=True),
           'fp8': SceneIndex(n, C, device=dev, coords=True, storage='fp8')}
    gen = torch.Generator(device=dev).manual_seed(0)
    anchors = torch.nn.functional.normalize(torch.randn(ANCHORS, C, generator=gen, device=dev), dim=1)
    rng = np.random.default_rng(0)
    for c in cs:
        rows = torch.nn.functional.normalize(torch.randn(len(c), C, generator=gen, device=dev), dim=1)
        for _ in range(6):                                   # seeded boxes
            ctr = c[rng.integers(len(c))]
            half = rng.integers(3, 12, 3)
            inside = torch.from_numpy(np.all(np.abs(c - ctr) <= half, 1)).to(dev)
            noise = 0.02 * torch.randn(int(inside.sum()), C, generator=gen, device=dev)
            rows[inside] = anchors[int(rng.integers(ANCHORS))] + noise
        cc = torch.from_numpy(c).to(dev)
        for i in idx.values():
            i.add(rows.half(), coords=cc)
    res['regions'] = {'rows': n, 'threshold': THR, 'R': R, 'reach': 1, 'runs': [],
                      'index_bytes': {k: n * row_bytes(k, C, coords=True) for k in idx}}
    for nq in a.nq:
        q = torch.cat([anchors, torch.nn.functional.normalize(
            torch.randn(max(0, nq - ANCHORS), C, generator=gen, device=dev), dim=1)])[:nq].half()
        t, out = alternate({k: (lambda i=i: i.regions(q, THR, max_regions=R, reach=1)) for k, i in idx.items()}, a.reps)
        r16, r8 = out['fp16'], out['fp8']
        r = {'nq': nq, 'sm_clock_now': smi('clocks.sm')}
        for k in idx:
            r[k] = {'ms_median': med(t[k]), 'ms_range': [min(t[k]), max(t[k])],
                    'regions': int(out[k].n_regions.sum())}
        top = lambda x: torch.stack([x.scene[:, 0], x.row[:, 0], x.size[:, 0]], 1)       # noqa: E731
        r['agreement'] = {'top_region': float((top(r16) == top(r8)).all(1).float().mean()),
                          'region_count_fp16': int(r16.n_regions.sum()), 'region_count_fp8': int(r8.n_regions.sum())}
        res['regions']['runs'].append(r)
        print(json.dumps(r), flush=True)
    res['time'] = time.strftime('%Y-%m-%d %H:%M:%S')
    with open(os.path.join(a.out, 'bench_scene_search_f8.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ('info', 'd2d_copy_GBps_read_plus_write', 'quantize_add_GBps_fp16_rows_in')}))


if __name__ == '__main__':
    main()
