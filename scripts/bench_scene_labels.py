"""Labelled scene index: ``SceneIndex.label``, ``class_counts`` and ``class_regions`` on the device, against the torch and
host routes a caller would otherwise take, in one run.

- label: 64 scenes of 196,000 seeded random rows (C = 768), K = 20 / 160 / 1,000 classes, fp16 and FP8 indices, against
  the torch route (1M-row chunks of ``rows @ vocab.T`` in fp16, then ``max(1)``).  Per arm the achieved rate of index read
  (TB/s) and of the product (2 N C K flop, TFLOP/s), and the agreement of the labels.
- class_counts over all K on the labelled fp16 index.
- class_regions: 64 ``synth.scene('config2_200k')`` scenes whose lowest two voxel layers are a floor-like class (millions
  of hits), with planted boxes of four more classes and seeded random rows elsewhere, K = 160, reach 1, R = 8, no
  threshold, at m = 1 (the floor) / 20 / 96; against the host route (labels -> ``nonzero`` -> a copy to the host -> SciPy
  connected components per scene and class) at m = 1 / 20.
- Peak device memory of each call above the index.

Arms alternate and are timed with CUDA events (medians and ranges over --reps after a warm-up).  The card's name, power
limit and SM clock are read in the same run.

    python scripts/bench_scene_labels.py --out DIR [--scenes 64] [--rows-per-scene 196000] [--reps 5]
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


def peak_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def torch_labels(idx, vocab, chunk=1 << 20):
    """the torch route: fp16 rows @ vocab.T per 1M-row chunk, max(1)"""
    n = idx.n_rows
    lab = torch.empty(n, dtype=torch.int64, device=idx.device)
    for a in range(0, n, chunk):
        lab[a:a + chunk] = (idx.rows[a:min(n, a + chunk)] @ vocab.T).max(1)[1]
    return lab


def host_regions(idx, classes):
    """labels -> nonzero -> host -> SciPy components per (scene, class): the number of regions"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    from scipy.spatial import cKDTree
    n = idx.n_rows
    lab = idx.row_label[:n]
    total = 0
    for c in classes:
        rows = torch.nonzero(lab == c).squeeze(1)
        rr = rows.cpu().numpy()
        sc = idx.row_scene[rows].cpu().numpy()
        xyz = idx.coords[rows, :3].cpu().numpy()
        cuts = np.r_[0, np.nonzero(np.diff(sc))[0] + 1, len(rr)]
        for a, b in zip(cuts[:-1], cuts[1:]):
            m = b - a
            if m == 0:
                continue
            pairs = cKDTree(xyz[a:b].astype(np.float64)).query_pairs(r=1.5, p=np.inf, output_type='ndarray')
            g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(m, m))
            total += connected_components(g, directed=False)[0]
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--scenes', type=int, default=64)
    ap.add_argument('--rows-per-scene', type=int, default=196_000)
    ap.add_argument('--channels', type=int, default=768)
    ap.add_argument('--K', type=int, nargs='+', default=[20, 160, 1000])
    ap.add_argument('--m', type=int, nargs='+', default=[1, 20, 96])
    ap.add_argument('--host-m', type=int, nargs='+', default=[1, 20])
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
           'note': 'seeded random rows, not OpenScene features'}

    # ---------------- label
    n = a.scenes * a.rows_per_scene
    idx = {'fp16': SceneIndex(n, C, device=dev), 'fp8': SceneIndex(n, C, device=dev, storage='fp8')}
    for s in range(a.scenes):
        gen = torch.Generator(device=dev).manual_seed(s)
        rows = (torch.randn(a.rows_per_scene, C, generator=gen, device=dev) * 0.05).half()
        for i in idx.values():
            i.add(rows)
    del rows
    row_bytes = {'fp16': 2 * C, 'fp8': C + 1}
    res['label'] = {'rows': n, 'scenes': a.scenes, 'runs': []}
    for K in a.K:
        vocab = torch.randn(K, C, generator=torch.Generator(device=dev).manual_seed(K), device=dev).half()
        arms = {k: (lambda i=i: i.label(vocab)) for k, i in idx.items()}
        arms['torch'] = lambda: torch_labels(idx['fp16'], vocab)
        t, out = alternate(arms, a.reps)
        r = {'K': K, 'sm_clock_now': smi('clocks.sm'), 'flop': 2 * n * C * K}
        for k in arms:
            ms = med(t[k])
            rb = row_bytes.get(k, 2 * C)
            r[k] = {'ms_median': ms, 'ms_range': [min(t[k]), max(t[k])],
                    'index_read_TBps': n * rb / (ms * 1e-3) / 1e12, 'TFLOPps': 2 * n * C * K / (ms * 1e-3) / 1e12}
        l16, l8 = idx['fp16'].row_label[:n], idx['fp8'].row_label[:n]
        r['agreement'] = {'fp16_vs_torch': float((l16 == out['torch']).float().mean()),
                          'fp8_vs_fp16': float((l8 == l16).float().mean())}
        r['peak_bytes_above_index'] = {k: peak_above(arms[k]) for k in ('fp16', 'fp8')}
        if K == max(a.K):
            tc, cnt = alternate({'counts': lambda: idx['fp16'].class_counts()}, a.reps)
            r['class_counts_all_K'] = {'ms_median': med(tc['counts']), 'ms_range': [min(tc['counts']), max(tc['counts'])],
                                       'peak_bytes': peak_above(lambda: idx['fp16'].class_counts()),
                                       'rows_counted': int(cnt['counts'].sum())}
        res['label']['runs'].append(r)
        print(json.dumps(r), flush=True)
    del idx
    torch.cuda.empty_cache()

    # ---------------- class regions with a floor-like class and planted objects
    K = 160
    cs = [synth.scene('config2_200k', seed=s)[:, 1:] for s in range(a.scenes)]
    n = sum(len(c) for c in cs)
    gen = torch.Generator(device=dev).manual_seed(0)
    vocab = torch.nn.functional.normalize(torch.randn(K, C, generator=gen, device=dev), dim=1)
    index = SceneIndex(n, C, device=dev, coords=True)
    rng = np.random.default_rng(0)
    for c in cs:
        rows = torch.nn.functional.normalize(torch.randn(len(c), C, generator=gen, device=dev), dim=1)
        floor = torch.from_numpy(c[:, 2] <= c[:, 2].min() + 1).to(dev)
        rows[floor] = vocab[0] + 0.02 * torch.randn(int(floor.sum()), C, generator=gen, device=dev)
        for _ in range(6):
            ctr = c[rng.integers(len(c))]
            half = rng.integers(3, 12, 3)
            inside = torch.from_numpy(np.all(np.abs(c - ctr) <= half, 1)).to(dev)
            rows[inside] = vocab[1 + int(rng.integers(4))] + 0.02 * torch.randn(int(inside.sum()), C, generator=gen,
                                                                              device=dev)
        index.add(rows.half(), coords=torch.from_numpy(c).to(dev))
    index.label(vocab.half())
    torch.cuda.synchronize()
    res['class_regions'] = {'rows': n, 'K': K, 'R': 8, 'reach': 1, 'runs': [],
                            'floor_rows': int(index.class_counts([0]).sum())}
    for m in a.m:
        classes = list(range(m))
        t, out = alternate({'device': lambda: index.class_regions(classes, max_regions=8)}, a.reps)
        hits = int(index.class_counts(classes, threshold=float('-inf')).sum())
        r = {'m': m, 'sm_clock_now': smi('clocks.sm'), 'hits': hits, 'ms_median': med(t['device']),
             'ms_range': [min(t['device']), max(t['device'])], 'regions': int(out['device'].n_regions.sum()),
             'peak_bytes_above_index': peak_above(lambda: index.class_regions(classes, max_regions=8))}
        if m in a.host_m:
            t0 = time.perf_counter()
            nreg = host_regions(index, classes)
            r['host_route'] = {'ms': (time.perf_counter() - t0) * 1e3, 'regions': int(nreg)}
        res['class_regions']['runs'].append(r)
        print(json.dumps(r), flush=True)
    res['time'] = time.strftime('%Y-%m-%d %H:%M:%S')
    with open(os.path.join(a.out, 'bench_scene_labels.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res['info']))


if __name__ == '__main__':
    main()
