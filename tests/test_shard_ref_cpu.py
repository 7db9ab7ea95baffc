"""The sharded index's merge restated in NumPy (tests/shard_ref.py) against one index holding every scene: per-shard
``search_ref`` / ``regions_ref`` results merged through the directory equal ``search_ref`` / ``regions_ref`` on the whole
score matrix in global order, over random assignments of scenes to ranks with out-of-order adds, cross-rank ties where
the higher rank holds the lower id, NaN / +-0 / inf scores, an empty rank, one scene, and 1-row scenes; and six mutated
rules fail.  Also: the directory logic over gloo (world 2, no GPU) raises the same error on both ranks, and the C ABI's
refusals of the merge entry points, in a child process."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import shard_ref
from tests.regions_ref import regions_ref
from tests.search_ref import search_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS_S = ('score', 'scene', 'row', 'scene_max', 'scene_argmax', 'scene_count')
FIELDS_R = ('score', 'scene', 'row', 'size', 'box_min', 'box_max', 'n_regions', 'hit_query', 'hit_scene', 'hit_row',
            'hit_score', 'hit_region')


def _eq(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float16:
        a = a.view(np.uint16)
    if b.dtype == np.float16:
        b = b.view(np.uint16)
    return a.shape == b.shape and np.array_equal(a, b)


def _scores(n, nq, rng):
    """coarse scores (many ties), planted NaN, +-0, +-inf and duplicated rows"""
    s = (np.round(rng.standard_normal((n, nq)) * 3) / 4).astype(np.float16)
    for r in rng.choice(n, min(n, 6), replace=False):
        s[r, rng.integers(nq)] = rng.choice(np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, -0.0], np.float16))
    if n > 4:
        s[n - 1] = s[0]
        s[n // 2] = s[1]
    return s


def _coords(off, rng, extent=6):
    out = []
    for a, b in zip(off[:-1], off[1:]):
        cells = rng.choice(max(extent, 3) ** 3, b - a, replace=False)
        out.append(np.stack(np.unravel_index(cells, (max(extent, 3),) * 3), 1))
    return np.concatenate(out).astype(np.int32)


def _assign(S, W, rng, empty_rank=None):
    """per rank the global ids in the order it adds them (shuffled)"""
    owner = rng.integers(0, W, S)
    if empty_rank is not None:
        owner[owner == empty_rank] = (empty_rank + 1) % W
    added = [list(rng.permutation(np.nonzero(owner == w)[0])) for w in range(W)]
    return added


def _search_case(s, off, added, k, thr, rule=None):
    sizes = np.diff(off)
    base = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    parts = []
    for ids_added in added:
        ids = shard_ref.local_ids(ids_added, rule)
        if not ids:
            parts.append((ids, shard_ref.empty_search(s.shape[1], k, thr is not None)))
            continue
        ls, loff, _ = shard_ref.shard(s, off, ids)
        parts.append((ids, search_ref(ls, loff, k, threshold=thr)))
    return shard_ref.merge_search(parts, base, rule)


def _regions_case(s, off, xyz, added, thr, R, reach, min_voxels, rule=None):
    sizes = np.diff(off)
    base = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    parts = []
    for ids_added in added:
        ids = shard_ref.local_ids(ids_added, rule)
        if not ids:
            parts.append((ids, shard_ref.empty_regions(s.shape[1], R)))
            continue
        ls, loff, lc = shard_ref.shard(s, off, ids, xyz)
        parts.append((ids, regions_ref(ls, lc, loff, thr, R, reach, min_voxels)))
    return shard_ref.merge_regions(parts, base, rule)


def _layout(S, rng, one_row=False):
    sizes = np.ones(S, np.int64) if one_row else rng.integers(1, 40, S)
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


@pytest.mark.parametrize('seed', range(8))
def test_search_merge_equals_the_single_index(seed):
    rng = np.random.default_rng(seed)
    S = [1, 2, 5, 13, 30, 7, 20, 9][seed]
    W = [1, 2, 3, 4, 8, 2, 5, 64][seed]
    off = _layout(S, rng, one_row=seed in (3, 5))
    nq = int(rng.integers(1, 7))
    s = _scores(int(off[-1]), nq, rng)
    added = _assign(S, W, rng, empty_rank=0 if W > 1 else None)
    for k in (1, 3, 32):
        for thr in (None, np.float32(0.25)):
            want = search_ref(s, off, k, threshold=None if thr is None else np.full(nq, thr, np.float32))
            got = _search_case(s, off, added, k, None if thr is None else np.full(nq, thr, np.float32))
            for f in FIELDS_S:
                assert _eq(got[f], want[f]), (f, k, thr)


def test_cross_rank_tie_goes_to_the_lower_id():
    """scene 3 on rank 1 and scene 7 on rank 0 hold the same row: the tie goes to id 3, not to rank 0"""
    rng = np.random.default_rng(1)
    off = _layout(10, rng)
    s = (rng.random((int(off[-1]), 2)) * 2 - 1).astype(np.float16)
    s[off[7]] = s[off[3]] = np.float16(60.0)
    added = [[7, 0, 2, 5, 9], [8, 3, 1, 4, 6]]
    got = _search_case(s, off, added, 1, None)
    assert (got['scene'][:, 0] == 3).all() and (got['row'][:, 0] == 0).all()
    for f in FIELDS_S:
        assert _eq(got[f], search_ref(s, off, 1)[f]), f


@pytest.mark.parametrize('seed', range(6))
def test_regions_merge_equals_the_single_index(seed):
    rng = np.random.default_rng(100 + seed)
    S, W = [1, 4, 9, 16, 6, 12][seed], [1, 2, 3, 4, 6, 3][seed]
    off = _layout(S, rng, one_row=seed == 4)
    xyz = _coords(off, rng)
    nq = int(rng.integers(1, 5))
    s = _scores(int(off[-1]), nq, rng)
    added = _assign(S, W, rng, empty_rank=1 if W > 2 else None)
    thr = np.full(nq, 0.25, np.float32)
    for R, reach, mv in ((1, 1, 1), (4, 2, 1), (32, 1, 3)):
        want = regions_ref(s, xyz, off, thr, R, reach, mv)
        got = _regions_case(s, off, xyz, added, thr, R, reach, mv)
        for f in FIELDS_R:
            assert _eq(got[f], want[f]), (f, R, reach, mv)


def _planted_case():
    """ties inside a rank added out of order, across ranks with the higher rank holding the lower id, and a -0 best"""
    rng = np.random.default_rng(7)
    off = np.concatenate([[0], np.cumsum([5, 6, 4, 7, 3, 20, 5, 6])]).astype(np.int64)
    n = int(off[-1])
    s = _scores(n, 3, rng)
    s[:, 2] = -1.0
    s[off[6], 2] = -0.0                          # the best of query 2 is a -0
    s[off[2] + 1, :2] = s[off[6] + 2, :2] = s[off[4], :2] = s[off[5] + 1, :2] = np.float16(40.0)
    s[off[5]:off[6], 1] = np.float16(35.0)       # a large region of scene 5, below scene 2's small one
    s[off[2]:off[2] + 1, 1] = np.float16(36.0)
    added = [[6, 5, 0, 1], [4, 2, 7, 3]]         # rank 1 holds id 2, rank 0 the higher ids 5 and 6, added out of order
    xyz = _coords(off, rng)
    xyz[off[5]:off[6]] = np.stack(np.unravel_index(np.arange(off[6] - off[5]), (5, 5, 5)), 1)   # one connected blob
    return s, off, xyz, added


@pytest.mark.parametrize('rule', ['tie_rank', 'local_ids', 'no_base', 'by_size', 'drop_sign', 'add_order'])
def test_mutated_rules_fail(rule):
    s, off, xyz, added = _planted_case()
    nq = s.shape[1]
    thr = np.full(nq, -2.0, np.float32)
    ok = True
    if rule != 'by_size':
        for k in (1, 2):
            want = search_ref(s, off, k, threshold=thr)
            got = _search_case(s, off, added, k, thr, rule)
            ok &= all(_eq(got[f], want[f]) for f in FIELDS_S)
    want = regions_ref(s, xyz, off, np.full(nq, 30.0, np.float32), 2, 1, 1)
    got = _regions_case(s, off, xyz, added, np.full(nq, 30.0, np.float32), 2, 1, 1, rule)
    ok &= all(_eq(got[f], want[f]) for f in FIELDS_R)
    if rule == 'drop_sign':
        want = search_ref(s, off, 1)
        got = _search_case(s, off, added, 1, None, rule)
        ok &= _eq(got['score'], want['score'])
    assert not ok, rule
    # the true rule passes the same case
    for thr_, k in ((thr, 2), (None, 1)):
        want, got = search_ref(s, off, k, threshold=thr_), _search_case(s, off, added, k, thr_)
        assert all(_eq(got[f], want[f]) for f in FIELDS_S)
    want = regions_ref(s, xyz, off, np.full(nq, 30.0, np.float32), 2, 1, 1)
    got = _regions_case(s, off, xyz, added, np.full(nq, 30.0, np.float32), 2, 1, 1)
    assert all(_eq(got[f], want[f]) for f in FIELDS_R)


# ------------------------------------------------------------------ the directory over gloo, no GPU

def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


CASES = {
    'ok': ([[0, 2], [1, 3]], [768, 768], ['fp16', 'fp16']),
    'empty_rank': ([[0, 1, 2], []], [512, 512], ['fp8', 'fp8']),
    'duplicate': ([[0, 1], [1, 2]], [768, 768], ['fp16', 'fp16']),
    'gap': ([[0, 1], [3]], [768, 768], ['fp16', 'fp16']),
    'width': ([[0], [1]], [768, 512], ['fp16', 'fp16']),
    'storage': ([[0], [1]], [768, 768], ['fp16', 'fp8']),
}


def _dir_worker(rank, world, port, ret):
    import datetime
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(minutes=2))
    from openscene_b200.search import build_directory
    out = {}
    try:
        for name, (ids, widths, storages) in CASES.items():
            mine = ids[rank]
            try:
                d = build_directory(mine, [10 + g for g in mine], [f's{g}' for g in mine], widths[rank], storages[rank])
                out[name] = ('ok', d.owner, d.local, d.base, d.names)
            except ValueError as e:
                out[name] = ('error', str(e))
        ret[rank] = out
    finally:
        dist.destroy_process_group()


def test_directory_refusals_are_the_same_on_every_rank():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dir_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    r0, r1 = ret[0], ret[1]
    assert r0 == r1
    assert r0['ok'] == ('ok', [0, 1, 0, 1], [0, 0, 1, 1], [0, 10, 21, 33], ['s0', 's1', 's2', 's3'])
    assert r0['empty_rank'][0] == 'ok' and r0['empty_rank'][1] == [0, 0, 0]
    assert r0['duplicate'][0] == 'error' and 'held twice' in r0['duplicate'][1]
    assert r0['gap'][0] == 'error' and 'id 2 is missing' in r0['gap'][1]
    assert r0['width'][0] == 'error' and 'widths' in r0['width'][1]
    assert r0['storage'][0] == 'error' and 'storages' in r0['storage'][1]


# ------------------------------------------------------------------ C ABI refusals

_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
out = {}
A = 1 << 20            # an aligned non-NULL placeholder: never dereferenced, every call is refused first
def rec(tag, rc):
    out[tag] = [rc, (L.osb_last_error() or b'').decode()]
def k(tag, n=10, nl=2, ng=4, rows=100, score=A, gid=A, key=A):
    rec(tag, L.osb_shard_keys(score, A, A, n, gid, nl, A, ng, rows, key, A, None))
k('k_n0', n=0); k('k_rows48', rows=1 << 48); k('k_local', nl=5); k('k_null', key=None); k('k_null_gid', gid=None)
k('k_misaligned', score=A + 1)
def m(tag, keys=A, world=2, nq=3, mm=8, win=A):
    rec(tag, L.osb_shard_merge(keys, world, nq, mm, win, None))
m('m_world0', world=0); m('m_world65', world=65); m('m_nq0', nq=0); m('m_nq_big', nq=65536); m('m_m0', mm=0)
m('m_m33', mm=33); m('m_null', keys=None); m('m_misaligned', win=A + 4)
def h(tag, n=10, world=2, nq=3, R=8, q=A, ws=A, wsb=1 << 30):
    rec(tag, L.osb_shard_hits(q, A, A, A, n, world, nq, R, A, A, A, ws, wsb, None))
h('h_world', world=65); h('h_nq', nq=0); h('h_R', R=33); h('h_n0', n=0); h('h_null', q=None); h('h_misaligned', q=A + 4)
h('h_short_ws', wsb=64); h('h_null_ws', ws=None); h('h_ws_misaligned', ws=A + 8)
out['ws0'] = [L.osb_shard_hits_workspace_bytes(0), '']
print('RESULT ' + json.dumps(out))
'''


def test_shard_refusals_happen_on_the_host_with_a_message():
    p = subprocess.run([sys.executable, '-c', _CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads([line for line in p.stdout.splitlines() if line.startswith('RESULT ')][-1][len('RESULT '):])
    assert res.pop('ws0')[0] == 0
    expect = {'k_n0': 'n=', 'k_rows48': '2^48', 'k_local': 'local scenes', 'k_null': 'NULL', 'k_null_gid': 'NULL',
              'k_misaligned': 'misaligned', 'm_world0': 'world=', 'm_world65': 'world=', 'm_nq0': 'nq=',
              'm_nq_big': 'nq=', 'm_m0': 'm=', 'm_m33': 'm=', 'm_null': 'NULL', 'm_misaligned': 'misaligned',
              'h_world': 'world=', 'h_nq': 'nq=', 'h_R': 'R=', 'h_n0': 'n_hits=', 'h_null': 'NULL',
              'h_misaligned': 'misaligned', 'h_short_ws': 'workspace', 'h_null_ws': 'workspace',
              'h_ws_misaligned': 'workspace'}
    assert sorted(res) == sorted(expect)
    for tag, (rc, err) in res.items():
        assert rc != 0, f"{tag}: accepted"
        assert expect[tag] in err, f"{tag}: {err!r}"
        assert err.startswith({'k': 'osb_shard_keys', 'm': 'osb_shard_merge', 'h': 'osb_shard_hits'}[tag[0]]), err
