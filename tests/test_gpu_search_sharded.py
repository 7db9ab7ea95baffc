"""The sharded scene index on the device (DESIGN.md, "Sharded index contract"): every output of ShardedSceneIndex.query and
.regions, on every rank, equals with torch.equal the output of one SceneIndex that adds the same scenes in ascending
global id, which each rank builds for itself from the same seeded scenes.

Runs: gloo world 2 with both ranks on cuda:0 (gloo stages CUDA tensors through the host: correctness only), gloo world 3
with one rank holding no scene, NCCL world 2 on cuda:0 / cuda:1 (skipped with fewer than two devices) and NCCL world 1
(both also check that query makes no host synchronisation, a side-stream run and outputs after the allocator's cache is
filled with sentinels), and groups of one rank against the bare index.  Scenes sit on tile edges, include 1-row scenes, and rows are
planted twice in scenes held by different ranks; scenes are added out of id order."""
import datetime
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

SIZES = [1, 127, 128, 129, 255, 300, 1, 64, 500, 2, 200, 257, 33]
PLANTS = [(7, 0, 3, 5), (9, 1, 2, 100), (11, 0, 5, 7), (12, 2, 8, 0)]     # (scene, row) <- (scene, row)


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _scenes(c, seed):
    """rows (fp16, scale 0.05) and distinct voxel coordinates per scene, the same on every rank"""
    g = torch.Generator().manual_seed(seed)
    rows = [(torch.randn(n, c, generator=g) * 0.05).half() for n in SIZES]
    for (s, r, s2, r2) in PLANTS:                 # duplicate rows in scenes that different ranks hold
        rows[s][r] = rows[s2][r2]
    rng = np.random.default_rng(seed)
    xyz = []
    for n in SIZES:
        cells = rng.choice(12 ** 3, n, replace=False)
        xyz.append(torch.from_numpy((np.stack(np.unravel_index(cells, (12,) * 3), 1) - 6).astype(np.int32)))
    return rows, xyz


def _owner(world, empty_last):
    rng = np.random.default_rng(world)
    ranks = world - 1 if empty_last else world
    owner = rng.integers(0, ranks, len(SIZES))
    owner[:ranks] = np.arange(ranks)
    owner[7], owner[3], owner[9], owner[2] = ranks - 1, 0, 0, ranks - 1     # planted pairs on different ranks
    return owner


def _h(t):
    return None if t is None else (t.view(torch.int16) if t.dtype == torch.float16 else t)


def _same(a, b, tag):
    for name, x, y in zip(a._fields, a, b):
        assert (x is None) == (y is None), (tag, name)
        if x is not None:
            assert x.dtype == y.dtype and torch.equal(_h(x), _h(y)), (tag, name)


def _build(rank, dev, c, storage, owner, group, rows, xyz):
    from openscene_b200.search import SceneIndex, ShardedSceneIndex
    N = sum(SIZES)
    ref = SceneIndex(N, c, device=dev, coords=True, storage=storage)
    for g in range(len(SIZES)):
        ref.add(rows[g].to(dev), name=f's{g}', coords=xyz[g].to(dev))
    idx = ShardedSceneIndex(N, c, process_group=group, device=dev, coords=True, storage=storage)
    mine = [g for g in range(len(SIZES)) if owner[g] == rank]
    for g in np.random.default_rng(rank + 17).permutation(mine):            # out of id order
        idx.add(rows[g].to(dev), int(g), name=f's{g}', coords=xyz[g].to(dev))
    return ref, idx


def _queries(nq, c, seed, dev):
    return torch.randn(nq, c, generator=torch.Generator().manual_seed(seed)).half().to(dev)


def _compare(rank, dev, c, storage, owner, group, full=True):
    rows, xyz = _scenes(c, seed=c + (1 if storage == 'fp8' else 0))
    ref, idx = _build(rank, dev, c, storage, owner, group, rows, xyz)
    idx.sync()
    assert idx.n_scenes == len(SIZES) and idx.names == [f's{g}' for g in range(len(SIZES))]
    assert [idx.owner(g) for g in range(len(SIZES))] == [int(o) for o in owner]
    tag = f"{storage} C={c}"
    for nq in ((1, 20, 96, 200) if full else (20,)):
        q = _queries(nq, c, nq, dev)
        for k in ((1, 8, 32) if full else (8,)):
            for thr in (None, 0.1):
                _same(idx.query(q, k=k, threshold=thr), ref.query(q, k=k, threshold=thr), f"{tag} query nq={nq} k={k}")
    q = _queries(24, c, 5, dev)
    for reach, R, mv in (((1, 1, 1), (2, 8, 1), (1, 32, 3), (2, 32, 1)) if full else ((1, 8, 1),)):
        for hits in (True, False):
            _same(idx.regions(q, 0.1, max_regions=R, reach=reach, min_voxels=mv, hits=hits),
                  ref.regions(q, 0.1, max_regions=R, reach=reach, min_voxels=mv, hits=hits),
                  f"{tag} regions reach={reach} R={R} min_voxels={mv} hits={hits}")
    q = _queries(100, c, 6, dev)                                              # two slices of queries
    _same(idx.regions(q, 0.12, max_regions=8, hits=True), ref.regions(q, 0.12, max_regions=8, hits=True),
          f"{tag} regions nq=100")
    return ref, idx


def _refusals(rank, world, dev, group):
    """group-level max_hits and status refusals, raised on every rank"""
    from openscene_b200.search import ShardedSceneIndex
    c = 512
    rows, xyz = _scenes(c, seed=3)
    owner = _owner(world, empty_last=False)
    ref, idx = _build(rank, dev, c, 'fp16', owner, group, rows, xyz)
    q = _queries(4, c, 9, dev)
    total = int(ref.query(q, k=1, threshold=0.1).scene_count.sum())
    local = int(idx.local.query(q, k=1, threshold=0.1).scene_count.sum()) if idx.local.n_scenes else 0
    if world > 1:
        assert local <= total - 1                                            # no rank alone exceeds the limit
    with pytest.raises(RuntimeError, match='over the group exceed max_hits'):
        idx.regions(q, 0.1, max_hits=total - 1)
    idx.regions(q, 0.1, max_hits=total)
    # duplicate coordinates on rank 0 only: every rank raises
    dup = ShardedSceneIndex(1000, c, process_group=group, device=dev, coords=True)
    xy = torch.zeros(50, 3, dtype=torch.int32, device=dev) if rank == 0 else \
        torch.stack([torch.arange(50, dtype=torch.int32, device=dev)] * 3, 1)
    dup.add(rows[5][:50].to(dev), rank, coords=xy)
    with pytest.raises(RuntimeError, match='share a voxel'):
        dup.regions(q, -1e4)


def _nccl_extras(rank, dev, ref, idx, c):
    q = _queries(40, c, 11, dev)
    base = idx.query(q, k=16, threshold=0.1)
    # outputs after the allocator's cache holds sentinels
    junk = torch.full((64 << 20,), 0x7f, dtype=torch.uint8, device=dev)
    del junk
    _same(idx.query(q, k=16, threshold=0.1), base, 'sentinel')
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        res = idx.query(q, k=16, threshold=0.1)
        reg = idx.regions(q, 0.1, max_regions=8, hits=True)
    torch.cuda.current_stream().wait_stream(side)
    _same(res, base, 'side stream')
    _same(reg, ref.regions(q, 0.1, max_regions=8, hits=True), 'side stream regions')
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r1 = idx.query(q, k=16, threshold=0.1)
        r2 = idx.query(q[:3], k=32)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _same(r1, base, 'sync-free query')
    _same(r2, ref.query(q[:3], k=32), 'sync-free query k=32')


def _worker(rank, world, backend, port, devices, empty_last):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device(devices[rank])
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(minutes=3))
    try:
        owner = _owner(world, empty_last)
        group = dist.group.WORLD
        if backend == 'nccl':
            for storage in ('fp16', 'fp8'):
                for c in (512, 768):
                    ref, idx = _compare(rank, dev, c, storage, owner, group, full=(c == 768))
            _nccl_extras(rank, dev, ref, idx, 768)
        elif empty_last:
            _compare(rank, dev, 768, 'fp16', owner, group, full=False)
            _compare(rank, dev, 512, 'fp8', owner, group, full=False)
        else:
            for storage in ('fp16', 'fp8'):
                for c in (512, 768):
                    _compare(rank, dev, c, storage, owner, group, full=(storage == 'fp16' and c == 768))
            # a group of one rank: every scene on it, against the bare index
            own = [dist.new_group([r]) for r in range(world)][rank]
            _compare(0, dev, 768, 'fp8', np.zeros(len(SIZES), np.int64), own, full=False)
        _refusals(rank, world, dev, group)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _spawn(world, backend, devices, empty_last=False):
    mp.spawn(_worker, args=(world, backend, _free_port(), devices, empty_last), nprocs=world, join=True)


def test_gloo_two_ranks_on_one_device():
    _spawn(2, 'gloo', ['cuda:0', 'cuda:0'])


def test_gloo_three_ranks_one_empty():
    _spawn(3, 'gloo', ['cuda:0'] * 3, empty_last=True)


def test_nccl_one_rank():
    """NCCL on one device: the checks of the NCCL run, host synchronisations included, over a group of one"""
    _spawn(1, 'nccl', ['cuda:0'])


def test_nccl_two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip(f"NCCL needs one device per rank: {torch.cuda.device_count()} visible")
    _spawn(2, 'nccl', ['cuda:0', 'cuda:1'])
