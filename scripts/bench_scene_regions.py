"""Scene regions: ``SceneIndex.regions`` against what a user writes today, on an index of 64 config2_200k scenes.

Data: each scene's voxel coordinates are ``synth.scene('config2_200k', seed=s)``.  Rows are planted: the voxels inside a
few seeded boxes per scene get one of four anchor embeddings plus noise, every other voxel a seeded random unit row.
Queries are the anchors followed by random unit rows.  Threshold 0.5, reach 1, R = 8.

Host arm: torch scores in 1M-row chunks (``rows @ q.T``), the threshold, ``nonzero``, a copy of the hits, their scores and
coordinates to the host, then per (scene, query) SciPy ``cKDTree.query_pairs(r=1, p=inf)`` and ``connected_components``,
and the per-query ranking.  The arms alternate and are timed with CUDA events (medians and ranges); ``query()`` at the
same nq is timed too, for the cost of the index read.  Agreement of the top regions is reported, not asserted (cuBLAS does
not round where the match kernel rounds, so hits near the threshold can differ).

    python scripts/bench_scene_regions.py --out DIR [--scenes 64] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

THR, R, ANCHORS = 0.5, 8, 4


def host_route(rows, coords, off, q, chunk=1 << 20):
    """-> per query a list of (score, scene, row, size, box_min, box_max), best first, and the hit count"""
    hits = []
    for a in range(0, rows.shape[0], chunk):
        s = rows[a:a + chunk] @ q.T
        nz = (s.float() >= THR).nonzero()
        hits.append((nz[:, 0] + a, nz[:, 1], s[nz[:, 0], nz[:, 1]]))
    r = torch.cat([h[0] for h in hits]).cpu().numpy()
    qq = torch.cat([h[1] for h in hits]).cpu().numpy()
    sc = torch.cat([h[2] for h in hits]).float().cpu().numpy()
    xyz = coords[torch.cat([h[0] for h in hits])].cpu().numpy()
    scene = np.searchsorted(off, r, side='right') - 1
    out = [[] for _ in range(q.shape[0])]
    order = np.lexsort((r, scene, qq))
    r, qq, sc, xyz, scene = r[order], qq[order], sc[order], xyz[order], scene[order]
    cuts = np.nonzero(np.diff(qq * (len(off) + 1) + scene))[0] + 1
    for lo, hi in zip(np.r_[0, cuts], np.r_[cuts, len(r)]):
        if hi == lo:
            continue
        n = hi - lo
        if n > 1:
            pairs = cKDTree(xyz[lo:hi]).query_pairs(r=1.5, p=np.inf, output_type='ndarray')
            lab = connected_components(coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(n, n)),
                                       directed=False)[1]
        else:
            lab = np.zeros(1, np.int64)
        for c in range(lab.max() + 1):
            m = np.nonzero(lab == c)[0] + lo
            b = m[np.lexsort((r[m], -sc[m]))[0]]
            out[qq[lo]].append((sc[b], scene[b], r[b] - off[scene[b]], len(m), xyz[m].min(0), xyz[m].max(0)))
    for j in range(len(out)):
        out[j].sort(key=lambda t: -t[0])
        out[j] = out[j][:R]
    return out, len(r)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def smi(fields):
    try:
        return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f'unavailable: {e}'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--scenes', type=int, default=64)
    ap.add_argument('--channels', type=int, default=768)
    ap.add_argument('--nq', type=int, nargs='+', default=[1, 20, 96])
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    os.makedirs(a.out, exist_ok=True)
    import __graft_entry__ as g
    g.build()
    from openscene_b200 import synth
    from openscene_b200.search import SceneIndex
    dev = torch.device('cuda:0')
    info = {'device': torch.cuda.get_device_name(0), 'power_limit_and_max_sm_clock': smi('power.limit,clocks.max.sm')}
    cs = [synth.scene('config2_200k', seed=s)[:, 1:] for s in range(a.scenes)]
    n_total = sum(len(c) for c in cs)
    idx = SceneIndex(n_total, a.channels, device=dev, coords=True)
    gen = torch.Generator(device=dev).manual_seed(0)
    anchors = torch.nn.functional.normalize(torch.randn(ANCHORS, a.channels, generator=gen, device=dev), dim=1)
    rng = np.random.default_rng(0)
    planted = 0
    for s, c in enumerate(cs):
        rows = torch.nn.functional.normalize(torch.randn(len(c), a.channels, generator=gen, device=dev), dim=1)
        for _ in range(6):                                   # seeded boxes
            ctr = c[rng.integers(len(c))]
            half = rng.integers(3, 12, 3)
            inside = torch.from_numpy(np.all(np.abs(c - ctr) <= half, 1)).to(dev)
            noise = 0.02 * torch.randn(int(inside.sum()), a.channels, generator=gen, device=dev)
            rows[inside] = anchors[int(rng.integers(ANCHORS))] + noise
            planted += int(inside.sum())
        idx.add(rows.half(), coords=torch.from_numpy(c).to(dev))
    coords = idx.coords[:n_total, :3]
    torch.cuda.synchronize()
    res = {'info': info, 'rows': n_total, 'scenes': a.scenes, 'channels': a.channels, 'threshold': THR, 'R': R,
           'reach': 1, 'planted_rows': planted, 'index_bytes': n_total * (2 * a.channels + 4 + 16), 'runs': []}
    med = lambda v: sorted(v)[len(v) // 2]                                      # noqa: E731
    for nq in a.nq:
        q = torch.cat([anchors, torch.nn.functional.normalize(
            torch.randn(max(0, nq - ANCHORS), a.channels, generator=gen, device=dev), dim=1)])[:nq].half()
        dev_fn = lambda: idx.regions(q, THR, max_regions=R, reach=1)            # noqa: E731
        host_fn = lambda: host_route(idx.rows[:n_total], coords, np.asarray(idx._off), q)   # noqa: E731
        query_fn = lambda: idx.query(q, k=R)                                    # noqa: E731
        dev_fn(); host_fn(); query_fn(); torch.cuda.synchronize()
        td, th, tq = [], [], []
        for _ in range(a.reps):                                                 # alternate the arms
            t, out_d = timed(dev_fn); td.append(t)
            t, (out_h, hits_h) = timed(host_fn); th.append(t)
            t, _ = timed(query_fn); tq.append(t)
        torch.cuda.reset_peak_memory_stats(); base = torch.cuda.memory_allocated()
        dev_fn(); torch.cuda.synchronize(); peak_d = torch.cuda.max_memory_allocated() - base
        n_reg = int(out_d.n_regions.sum())
        cnt = int(idx.query(q, k=1, threshold=THR).scene_count.sum())
        top_d = [(int(out_d.scene[j, 0]), int(out_d.row[j, 0]), int(out_d.size[j, 0])) for j in range(nq)]
        top_h = [(int(o[0][1]), int(o[0][2]), int(o[0][3])) if o else (-1, -1, 0) for o in out_h]
        r = {'nq': nq, 'device_ms_median': med(td), 'device_ms_range': [min(td), max(td)],
             'host_ms_median': med(th), 'host_ms_range': [min(th), max(th)],
             'query_ms_median': med(tq), 'query_ms_range': [min(tq), max(tq)],
             'hits_device': cnt, 'hits_host': hits_h, 'regions_device': n_reg,
             'device_peak_bytes_above_index': peak_d, 'sm_clock_now': smi('clocks.sm'),
             'top_region_agreement': float(np.mean([x == y for x, y in zip(top_d, top_h)]))}
        res['runs'].append(r)
        print(json.dumps(r), flush=True)
    res['time'] = time.strftime('%Y-%m-%d %H:%M:%S')
    with open(os.path.join(a.out, 'bench_scene_regions.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({'info': info, 'rows': n_total, 'planted_rows': planted}))


if __name__ == '__main__':
    main()
