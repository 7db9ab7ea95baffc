"""Scene search: the device search (openscene_b200.search) against the torch route, on an index of 64 config2_200k-sized
scenes (seeded random fp16 rows; the cost of a search does not depend on how the rows were made).

The torch route: 1M-row chunks of ``rows @ q.T``, ``topk`` per chunk and a merge, and ``scatter_reduce('amax')`` per
scene.  The two arms alternate and are timed with CUDA events.  Also measured in the same run: a device-to-device copy of
1 GiB, for the achieved bandwidth of the index read.  Top-1 agreement between the arms is reported, not asserted (cuBLAS
does not round where the matching kernels round).

    python scripts/bench_scene_search.py --out DIR [--scenes 64] [--rows-per-scene 196000] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def torch_route(rows, row_scene, n_scenes, q, k, chunk=1 << 20):
    best_v, best_i = None, None
    for a in range(0, rows.shape[0], chunk):
        s = rows[a:a + chunk] @ q.T                          # [chunk, nq] fp16
        v, i = torch.topk(s, min(k, s.shape[0]), dim=0)
        i = i + a
        if best_v is not None:
            v, j = torch.topk(torch.cat([best_v, v]), k, dim=0)
            i = torch.gather(torch.cat([best_i, i]), 0, j)
        best_v, best_i = v, i
        sm = torch.full((n_scenes, q.shape[0]), float('-inf'), dtype=torch.float16, device=rows.device)
        sm = sm.scatter_reduce(0, row_scene[a:a + chunk].long()[:, None].expand_as(s), s, 'amax')
        smax = sm if a == 0 else torch.maximum(smax, sm)
    return best_v.T, best_i.T, smax


def timed(fn, reps):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return times, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--scenes', type=int, default=64)
    ap.add_argument('--rows-per-scene', type=int, default=196_000)
    ap.add_argument('--channels', type=int, default=768)
    ap.add_argument('--k', type=int, default=32)
    ap.add_argument('--nq', type=int, nargs='+', default=[1, 20, 96])
    ap.add_argument('--reps', type=int, default=7)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    os.makedirs(a.out, exist_ok=True)
    import __graft_entry__ as g
    g.build()
    from openscene_b200.search import SceneIndex
    dev = torch.device('cuda:0')
    info = {'device': torch.cuda.get_device_name(0)}
    try:
        info['power_limit'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        info['power_limit'] = f'unavailable: {e}'
    n_total = a.scenes * a.rows_per_scene
    idx = SceneIndex(n_total, a.channels, device=dev)
    for s in range(a.scenes):
        gen = torch.Generator(device=dev).manual_seed(s)
        idx.add((torch.randn(a.rows_per_scene, a.channels, generator=gen, device=dev) * 0.05).half())
    torch.cuda.synchronize()
    index_bytes = n_total * (2 * a.channels + 4)
    src = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    copy_t, _ = timed(lambda: dst.copy_(src), a.reps)
    copy_gbs = 2 * src.numel() / (sorted(copy_t)[len(copy_t) // 2] * 1e-3) / 1e9
    del src, dst
    res = {'info': info, 'rows': n_total, 'scenes': a.scenes, 'channels': a.channels, 'k': a.k,
           'index_bytes': index_bytes, 'd2d_copy_GBps_read_plus_write': copy_gbs, 'runs': []}
    for nq in a.nq:
        gen = torch.Generator(device=dev).manual_seed(1000 + nq)
        q = torch.randn(nq, a.channels, generator=gen, device=dev).half()
        dev_fn = lambda: idx.query(q, k=a.k)                                   # noqa: E731
        tor_fn = lambda: torch_route(idx.rows[:n_total], idx.row_scene[:n_total], a.scenes, q, a.k)   # noqa: E731
        dev_fn(); tor_fn(); torch.cuda.synchronize()
        td, tt = [], []
        for _ in range(a.reps):                       # alternate the arms
            t, out_d = timed(dev_fn, 1); td += t
            t, out_t = timed(tor_fn, 1); tt += t
        torch.cuda.reset_peak_memory_stats(); base = torch.cuda.memory_allocated()
        dev_fn(); torch.cuda.synchronize(); peak_d = torch.cuda.max_memory_allocated() - base
        torch.cuda.reset_peak_memory_stats(); base = torch.cuda.memory_allocated()
        tor_fn(); torch.cuda.synchronize(); peak_t = torch.cuda.max_memory_allocated() - base
        grow_d = (torch.tensor(idx._off, device=dev)[out_d.scene[:, 0]] + out_d.row[:, 0])
        agree = float((grow_d == out_t[1][:, 0]).float().mean())
        smax_agree = float((out_d.scene_max == out_t[2]).float().mean())
        med = lambda v: sorted(v)[len(v) // 2]                                  # noqa: E731
        r = {'nq': nq, 'device_ms_median': med(td), 'device_ms_range': [min(td), max(td)],
             'torch_ms_median': med(tt), 'torch_ms_range': [min(tt), max(tt)],
             'device_index_read_GBps': index_bytes / (med(td) * 1e-3) / 1e9,
             'device_peak_bytes': peak_d, 'torch_peak_bytes': peak_t,
             'top1_row_agreement': agree, 'scene_max_agreement': smax_agree}
        res['runs'].append(r)
        print(json.dumps(r), flush=True)
    res['time'] = time.strftime('%Y-%m-%d %H:%M:%S')
    with open(os.path.join(a.out, 'bench_scene_search.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({'info': info, 'd2d_copy_GBps_read_plus_write': copy_gbs}))


if __name__ == '__main__':
    main()
