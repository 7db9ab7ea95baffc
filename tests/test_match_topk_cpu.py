"""tests/topk_ref.py without a GPU: the top-k ordering rule on hand-built rows (ties, +-0, +-inf, one NaN, all NaN, K = 1,
k > K refused), against torch.topk on rows without ties or NaN, against torch's CPU ``max(1)[1]`` for k = 1, its torch
version against the NumPy one, and two mutated rules (ties to the higher column; NaN last) that must fail.  The C ABI of
osb_match_topk / osb_match_ensemble_topk in a child process: each refusal with otherwise valid arguments and NULL buffers,
so that nothing could be launched, returns non-zero with a message naming the argument."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import topk_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN, INF = float('nan'), float('inf')

# (row, k, expected labels)
CASES = [
    ([1.0, 3.0, 3.0, 2.0], 3, [1, 2, 3]),                       # tie: the lower column first
    ([0.0, -0.0, 0.0, -1.0], 3, [0, 1, 2]),                     # -0 == +0
    ([-0.0, 0.0, -1.0], 2, [0, 1]),
    ([5.0, INF, -INF, 65504.0], 4, [1, 3, 0, 2]),               # inf above every finite value, -inf last
    ([-INF, -INF, -INF], 2, [0, 1]),
    ([1.0, NAN, 7.0, 2.0], 2, [1, 2]),                          # one NaN ranks first
    ([NAN, NAN, NAN, NAN], 3, [0, 1, 2]),                       # all NaN: ascending columns
    ([2.0, NAN, INF, NAN, 2.0], 5, [1, 3, 2, 0, 4]),
    ([-3.5], 1, [0]),                                           # K = 1
    ([NAN], 1, [0]),
]


def _row(v):
    return np.array([v], dtype=np.float16)


@pytest.mark.parametrize('row,k,want', CASES)
def test_hand_built_rows(row, k, want):
    lab, sc = R.topk(_row(row), k)
    assert lab.tolist() == [want]
    got = sc[0].astype(np.float64)
    ref = np.array(row, dtype=np.float16)[want].astype(np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[~np.isnan(got)], ref[~np.isnan(ref)])
    # the scores keep their own bits (the sign of a zero included)
    assert np.array_equal(sc[0].view(np.uint16)[~np.isnan(got)], np.array(row, dtype=np.float16)[want].view(np.uint16)[~np.isnan(ref)])
    tl, ts = R.topk_torch(torch.from_numpy(_row(row)), k)
    assert tl.tolist() == [want]
    assert np.array_equal(ts.numpy().view(np.uint16), sc.view(np.uint16))


def test_k_outside_1_to_K_is_refused():
    for k in (0, 4):
        with pytest.raises(ValueError):
            R.topk(_row([1.0, 2.0, 3.0]), k)
        with pytest.raises(ValueError):
            R.topk_torch(torch.from_numpy(_row([1.0, 2.0, 3.0])), k)


def test_agrees_with_torch_topk_without_ties_or_nan():
    g = np.random.RandomState(0)
    for K in (1, 2, 9, 96, 97, 500):
        for _ in range(20):
            s = g.permutation(np.arange(-K // 2, K - K // 2))[None].astype(np.float16) / np.float16(4)   # distinct values
            for k in sorted({1, min(3, K), min(8, K)}):
                lab, sc = R.topk(s, k)
                t = torch.from_numpy(s).float().topk(k, dim=1)
                assert np.array_equal(lab, t.indices.numpy()) and np.array_equal(sc.astype(np.float32), t.values.numpy())


def _messy(n, K, g):
    """few distinct values (ties everywhere), +-0, +-inf and NaN sprinkled in"""
    s = g.choice(np.array([-2, -1, -0.0, 0.0, 0.5, 1, 3, INF, -INF, NAN], dtype=np.float16), size=(n, K),
                 p=[.1, .15, .1, .1, .15, .15, .1, .05, .05, .05])
    s[0] = np.nan
    return s


def test_first_column_is_torch_cpu_argmax():
    """k = 1: the first NaN of a row if it holds one, else the first maximum (torch's CPU ``x.float().max(1)[1]``)"""
    g = np.random.RandomState(1)
    for K in (1, 2, 7, 96, 300):
        s = _messy(200, K, g)
        lab, _ = R.topk(s, 1)
        assert np.array_equal(lab[:, 0], torch.from_numpy(s).float().max(1)[1].numpy())


def test_torch_version_equals_numpy_version():
    g = np.random.RandomState(2)
    for K in (1, 3, 96, 481):
        s = _messy(300, K, g)
        cols = np.stack([g.permutation(10 * K)[:K] for _ in range(300)])      # merged slices: columns in any order
        for k in sorted({1, min(3, K), min(8, K)}):
            for c in (None, cols):
                lab, sc = R.topk(s, k, c)
                tl, ts = R.topk_torch(torch.from_numpy(s), k, None if c is None else torch.from_numpy(c))
                assert np.array_equal(tl.numpy(), lab) and np.array_equal(ts.numpy().view(np.uint16), sc.view(np.uint16))


def test_slices_merge_to_the_whole():
    g = np.random.RandomState(3)
    s = _messy(100, 1000, g)
    for k in (1, 5, 8):
        parts = [R.topk(s[:, j:j + 96], k) for j in range(0, 1000, 96) if s[:, j:j + 96].shape[1] >= k]
        cols = np.concatenate([p[0] + j for p, j in zip(parts, range(0, 1000, 96))], 1)
        merged = R.topk(np.concatenate([p[1] for p in parts], 1), k, cols)
        assert np.array_equal(merged[0], R.topk(s, k)[0])


def _ties_high(s, k):
    K = s.shape[1]
    lab, sc = R.topk(s[:, ::-1], k)
    return K - 1 - lab, sc


def _nan_last(s, k):
    v = s.astype(np.float64)
    nan = np.isnan(v)
    order = np.lexsort((np.broadcast_to(np.arange(s.shape[1]), s.shape), -np.where(nan, 0, v) - 0.0, nan), axis=-1)[:, :k]
    return order, np.take_along_axis(s, order, 1)


@pytest.mark.parametrize('mutant', [_ties_high, _nan_last])
def test_mutated_rules_fail(mutant):
    wrong = 0
    for row, k, want in CASES:
        lab, _ = mutant(_row(row), k)
        wrong += lab.tolist() != [want]
    assert wrong >= 2


# ------------------------------------------------------------------------------------------------ C ABI refusals
_CHILD = r'''
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
host = ctypes.create_string_buffer(64)          # a non-NULL pointer that is never launched on
H = ctypes.addressof(host)
out = {}
def run(name, *args):
    return [getattr(L, name)(*args), (L.osb_last_error() or b'').decode()]
def topk(c=768, k_text=1203, topk=5, n_vox=10, n_pts=10, text=H, label=H, feat=None):
    return run('osb_match_topk', feat, 0, n_vox, c, None, n_pts, text, k_text, 0, topk, None, label, None, None)
def ens(c=512, k_text=1203, topk=5, n_vox=10, n_pts=10, text=H, label=H, feat=None):
    return run('osb_match_ensemble_topk', feat, feat, n_vox, c, None, n_pts, feat, feat, text, k_text, topk, None, label,
               None, None)
for name, f in (('topk', topk), ('ensemble', ens)):
    out[name + ':c=600'] = f(c=600)
    out[name + ':c=0'] = f(c=0)
    out[name + ':k_text=0'] = f(k_text=0)
    out[name + ':k_text=1048577'] = f(k_text=1048577)
    out[name + ':k_text=-5'] = f(k_text=-5)
    out[name + ':topk=0'] = f(topk=0)
    out[name + ':topk=9'] = f(topk=9)
    out[name + ':topk>K'] = f(k_text=2, topk=3)
    out[name + ':n_vox=0'] = f(n_vox=0)
    out[name + ':n_pts=-1'] = f(n_pts=-1)
    out[name + ':text NULL'] = f(text=None)
    out[name + ':label NULL'] = f(label=None)
    out[name + ':features NULL'] = f()
print('RESULT ' + json.dumps(out))
'''

_WANT = {'c=600': 'feature width 600', 'c=0': 'feature width 0', 'k_text=0': 'K_text=0 outside 1..1048576',
         'k_text=1048577': 'K_text=1048577 outside', 'k_text=-5': 'K_text=-5 outside', 'topk=0': 'topk=0 outside',
         'topk=9': 'topk=9 outside 1..min(8', 'topk>K': 'topk=3 outside 1..min(8, K_text=2)', 'n_vox=0': 'n_vox=0',
         'n_pts=-1': 'n_pts=-1', 'text NULL': 'NULL text', 'label NULL': 'NULL label', 'features NULL': 'NULL features'}


def test_abi_refuses_each_bad_argument_with_a_message_naming_it():
    p = subprocess.run([sys.executable, '-c', _CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
    assert len(res) == 2 * len(_WANT)
    for key, (rc, err) in res.items():
        name, case = key.split(':', 1)
        fn = 'osb_match_topk' if name == 'topk' else 'osb_match_ensemble_topk'
        assert rc != 0 and err.startswith(fn + ':') and _WANT[case] in err, (key, rc, err)
