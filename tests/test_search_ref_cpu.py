"""The scene search restatement (tests/search_ref.py) against torch, on planted edge cases and against mutated rules; and
the C ABI's refusals of osb_search, in a child process (no GPU: they happen before any CUDA call)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.search_ref import search_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _eq(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float16:
        return np.array_equal(a.view(np.uint16), b.view(np.uint16))
    return np.array_equal(a, b)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_against_torch_topk_and_scatter_reduce_on_tie_free_data(seed):
    rng = np.random.default_rng(seed)
    n, nq, k = 3000, 5, 7
    bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    finite = bits[((bits & 0x7fff) < 0x7c00) & (bits != 0x8000)]          # every finite value once (no -0)
    s = rng.choice(finite, n * nq, replace=False).view(np.float16).reshape(n, nq)
    assert len(np.unique(s.view(np.uint16))) == n * nq
    off = np.concatenate([[0], np.sort(rng.choice(np.arange(1, n), 40, replace=False)), [n]])
    r = search_ref(s, off, k, threshold=0.0)
    t = torch.from_numpy(s.astype(np.float32))
    tv, ti = torch.topk(t, k, dim=0)
    assert _eq(r['score'].T.astype(np.float32), tv.numpy())
    scene_of = np.repeat(np.arange(len(off) - 1), np.diff(off))
    assert np.array_equal(r['scene'].T, scene_of[ti.numpy()])
    assert np.array_equal(r['row'].T, ti.numpy() - off[scene_of[ti.numpy()]])
    idx = torch.from_numpy(scene_of).long()[:, None].expand(n, nq)
    amax = torch.full((len(off) - 1, nq), -np.inf).scatter_reduce(0, idx, t, 'amax', include_self=True)
    assert _eq(r['scene_max'].astype(np.float32), amax.numpy())
    for sc in range(len(off) - 1):
        blk = s[off[sc]:off[sc + 1]].astype(np.float32)
        assert np.array_equal(r['scene_argmax'][sc], blk.argmax(0))
        assert np.array_equal(r['scene_count'][sc], (blk >= 0).sum(0))


def _planted():
    nan, inf = np.float16(np.nan), np.float16(np.inf)
    col = np.array([1, 3, 3, -0.0, 0.0, nan, inf, -inf, 3, nan, 0.0, -0.0, 2], np.float16)
    off = np.array([0, 2, 5, 9, 13])
    return col[:, None], off


def test_planted_ties_zeros_nan_inf_and_padding():
    s, off = _planted()
    r = search_ref(s, off, 12, threshold=0.0)
    # inf (row 6), then the three 3s by row (1, 2, 8), then 2, 1, then the four zeros by row, then -inf; NaN never
    assert list(r['score'][0, :11].astype(np.float32)) == [np.inf, 3, 3, 3, 2, 1, 0, 0, 0, 0, -np.inf]
    assert np.array_equal(r['scene'][0, :11], [2, 0, 1, 2, 3, 0, 1, 1, 3, 3, 2])
    assert np.array_equal(r['row'][0, :11], [1, 1, 0, 3, 3, 0, 1, 2, 1, 2, 2])
    assert np.isneginf(r['score'][0, 11]) and r['scene'][0, 11] == -1 and r['row'][0, 11] == -1
    # scene 1 = [3, -0, +0]: max 3 at row 0; scene 3 = [nan, 0, -0, 2]
    assert np.array_equal(r['scene_argmax'][:, 0], [1, 0, 1, 3])
    # the zero kept its sign: a scene of only (-0, +0) keeps the first (-0)
    r2 = search_ref(np.array([[-0.0], [0.0]], np.float16), [0, 2], 2)
    assert r2['scene_max'][0, 0].view(np.uint16) == 0x8000 and r2['scene_argmax'][0, 0] == 0
    assert np.array_equal(r['scene_count'][:, 0], [2, 3, 2, 3])
    allnan = search_ref(np.full((3, 1), np.nan, np.float16), [0, 3], 2, threshold=-np.inf)
    assert np.isneginf(allnan['scene_max'][0, 0]) and allnan['scene_argmax'][0, 0] == -1
    assert allnan['scene_count'][0, 0] == 0 and (allnan['row'] == -1).all()
    nothr = search_ref(s, off, 2, threshold=np.nan)
    assert (nothr['scene_count'] == 0).all()


@pytest.mark.parametrize('rule', ['nan_first', 'tie_high', 'neg_zero_low', 'boundary'])
def test_mutated_rules_fail(rule):
    s, off = _planted()
    good = search_ref(s, off, 12, threshold=0.0)
    bad = search_ref(s, off, 12, threshold=0.0, rule=rule)
    assert not all(_eq(good[key], bad[key]) for key in ('score', 'scene', 'row', 'scene_max', 'scene_argmax',
                                                        'scene_count')), rule


_CHILD = r'''
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
out = {}
A = 1 << 20            # a 16-byte aligned non-NULL placeholder: never dereferenced, every call is refused first
def off(*v):
    return (C.I64 * len(v))(*v)
def run(tag, c=768, n=10, S=1, offs=None, nq=4, k=2, rows=A, ws_bytes=1 << 30, count=None, thr=None, out_p=A):
    offs = offs if offs is not None else off(0, n)
    r = L.osb_search(rows, A, n, c, offs, A, S, A, nq, k, thr, out_p, A, A, A, A, count, A, ws_bytes, None)
    out[tag] = [r, (L.osb_last_error() or b'').decode()]
run('width', c=640)
run('nq0', nq=0); run('nq97', nq=97); run('k0', k=0); run('k33', k=33)
run('n0', n=0, offs=off(0, 0)); run('S0', S=0, offs=off(0))
run('big', n=1 << 31, offs=off(0, 1 << 31))
run('start', S=2, offs=off(1, 5, 10)); run('end', S=2, offs=off(0, 5, 9)); run('flat', S=2, offs=off(0, 0, 10))
run('down', S=3, offs=off(0, 6, 4, 10))
run('null_rows', rows=None); run('null_out', out_p=None); run('count_no_thr', count=A)
run('misaligned', rows=A + 2)
run('ws', ws_bytes=8)
out['ws_bytes'] = [L.osb_search_workspace_bytes(3, 4, 2), L.osb_search_workspace_bytes(3, 97, 2),
                   L.osb_search_workspace_bytes(0, 4, 2), L.osb_search_workspace_bytes(3, 4, 33)]
print('RESULT ' + json.dumps(out))
'''


def test_search_refusals_happen_on_the_host_with_a_message():
    p = subprocess.run([sys.executable, '-c', _CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
    ws = res.pop('ws_bytes')
    assert ws[0] > 0 and ws[1:] == [0, 0, 0]
    expect = {'width': 'width', 'nq0': 'nq', 'nq97': 'nq', 'k0': 'k=', 'k33': 'k=', 'n0': 'N=', 'S0': 'scenes',
              'big': 'N=', 'start': 'offsets', 'end': 'offsets', 'flat': 'strictly', 'down': 'strictly',
              'null_rows': 'NULL', 'null_out': 'NULL', 'count_no_thr': 'threshold', 'misaligned': 'aligned',
              'ws': 'workspace'}
    for tag, (rc, err) in res.items():
        assert rc != 0, f"{tag}: accepted"
        assert expect[tag] in err, f"{tag}: {err!r}"
