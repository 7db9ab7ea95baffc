"""Sharded scene search (DESIGN.md, "Sharded index contract"), run under torch.distributed.run:

    python -m torch.distributed.run --nproc_per_node N scripts/bench_scene_search_sharded.py --out DIR

Each rank holds --scenes scenes of --rows-per-scene seeded rows (64 fp16 or 128 FP8 scenes of 196,000 rows, the
workloads of bench_scene_search*.py), global ids rank, rank + N, ...  Per nq (k = 32) it times, with CUDA events and in
turn: the rank's local search (SceneIndex.query on its shard), the sharded query end to end, and their difference (the
collective plus the merge).  Regions: the same rows with distinct voxel coordinates, threshold 4.0 (a few thousand
hits per query), R = 8.  Separately, on one device, the merge kernel alone at world 8 on synthetic sorted lists.  Rank 0 writes one JSON file with the card,
its power limit and SM clock beside every number."""
import argparse
import datetime
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bench_scene_search_f8 import alternate, med, search_rows, smi, timed   # noqa: E402


def merge_alone(dev, world=8, nq=96, m=32, reps=200):
    from openscene_b200 import _cabi as C
    g = torch.Generator(device=dev).manual_seed(0)
    keys = torch.randint(1, 2 ** 62, (world, nq, m), generator=g, device=dev).sort(dim=2, descending=True).values
    win = torch.empty((nq, m), dtype=torch.int64, device=dev)

    def run():
        for _ in range(reps):
            C.call('osb_shard_merge', C.ptr(keys), world, nq, m, C.ptr(win), C.stream_ptr())
    run()
    dt, _ = timed(run)
    flat = keys.permute(1, 0, 2).reshape(nq, world * m)
    want = flat.topk(m, dim=1).values
    assert torch.equal(flat.gather(1, win), want), "merge disagrees with topk"
    return dt / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--storage', choices=['fp16', 'fp8'], default='fp16')
    ap.add_argument('--scenes', type=int, default=None, help='per rank (default 64 fp16, 128 fp8)')
    ap.add_argument('--rows-per-scene', type=int, default=196_000)
    ap.add_argument('--nq', type=int, nargs='+', default=[1, 20, 96])
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    from openscene_b200.search import ShardedSceneIndex
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    dev = torch.device('cuda', int(os.environ.get('LOCAL_RANK', 0)))
    torch.cuda.set_device(dev)
    dist.init_process_group('nccl', rank=rank, world_size=world, timeout=datetime.timedelta(minutes=10))
    S = a.scenes or (64 if a.storage == 'fp16' else 128)
    n, c = a.rows_per_scene, 768
    idx = ShardedSceneIndex(S * n, c, device=dev, coords=True, storage=a.storage)
    rng = np.random.default_rng(rank)
    for j in range(S):
        g = rank + world * j
        cells = torch.from_numpy(rng.choice(160 ** 3, n, replace=False).astype(np.int64)).to(dev)
        xyz = torch.stack([cells // 25600, cells // 160 % 160, cells % 160], 1) - 80
        idx.add(search_rows(g, n, c, dev), g, coords=xyz)
    idx.sync()
    out = dict(card=smi('name'), power_limit_and_max_sm_clock=smi('power.limit,clocks.max.sm'),
               sm_clock_now=smi('clocks.sm'), world=world, storage=a.storage, scenes_per_rank=S, rows_per_scene=n,
               rows_per_rank=S * n, k=32, search={}, regions={})
    for nq in a.nq:
        q = (torch.randn(nq, c, generator=torch.Generator(device=dev).manual_seed(nq), device=dev)).half()
        t, _ = alternate({'local': lambda: idx.local.query(q, k=32),
                          'sharded': lambda: idx.query(q, k=32)}, a.reps)
        out['search'][nq] = dict(local_ms=med(t['local']), end_to_end_ms=med(t['sharded']),
                                 collective_and_merge_ms=med(t['sharded']) - med(t['local']))
        t, res = alternate({'sharded': lambda: idx.regions(q, 4.0, max_regions=8)}, a.reps)
        out['regions'][nq] = dict(end_to_end_ms=med(t['sharded']),
                                  regions_found=int((res['sharded'].size > 0).sum()))
    out['merge_kernel_world8_nq96_m32_us'] = merge_alone(dev)
    out['sm_clock_after'] = smi('clocks.sm')
    if rank == 0:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f'sharded_{a.storage}_world{world}.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
