"""The pooling restatement (tests/pool_ref.py) checked without a GPU: against the oracle's sum / average pooling bit for bit,
against torch's dense max / average pooling and their autograd on fully occupied grids (offsets and strides checked
independently of the sparse machinery), on hand-built tie, NaN, +-inf and +-0 windows, and against mutated restatements
that must be caught."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import me_cpu
from openscene_b200 import synth
from tests import pool_ref as P


def _nbr(om, ts_in, ts_out, ks, dil=1):
    maps = om.kernel_map(ts_in, ts_out, ks, dil)
    nbr = np.full((len(maps), len(om.coords[ts_out])), -1, np.int64)
    for k, (ii, oo) in enumerate(maps):
        nbr[k, oo.numpy()] = ii.numpy()
    return nbr


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize('ks,stride,dil', [(2, 2, 1), (3, 1, 1), (3, 2, 1), (3, 1, 2), (1, 2, 1)])
def test_sum_and_avg_equal_the_oracle_bit_for_bit(ks, stride, dil):
    cl = synth.random_cloud(1500, 20, seed=4, batch=2)
    x = torch.randn(len(cl), 7, generator=torch.Generator().manual_seed(ks + stride), dtype=torch.float32) * 3
    om = me_cpu.CoordinateManager(cl)
    xo = me_cpu.SparseTensor(x, coordinate_manager=om)
    ts_out = om.stride(1, stride) if stride > 1 else 1
    nbr = _nbr(om, 1, ts_out, ks, dil)
    for mode, cls in ((P.SUM, me_cpu.MinkowskiSumPooling), (P.AVG, me_cpu.MinkowskiAvgPooling)):
        y = cls(kernel_size=ks, stride=stride, dilation=dil, dimension=3)(xo).F.numpy()
        out, cnt, _ = P.pool_fwd(x.numpy(), nbr, mode)
        assert np.array_equal(_bits(out), _bits(y)), mode


def _dense_case(seed, B=2, C=3, S=8):
    """fully occupied B x S^3 grid, distinct values: sparse rows (oracle order) <-> dense [B, C, S, S, S]"""
    g = torch.Generator().manual_seed(seed)
    dense = (torch.randperm(B * C * S ** 3, generator=g).float() / 7).reshape(B, C, S, S, S)
    b, xx, yy, zz = np.meshgrid(np.arange(B), np.arange(S), np.arange(S), np.arange(S), indexing='ij')
    coords = np.stack([b, xx, yy, zz], -1).reshape(-1, 4)
    feats = dense.permute(0, 2, 3, 4, 1).reshape(-1, C)
    return dense, coords, feats


def _to_dense(rows, coords, ts, B, C, S):
    out = torch.full((B, C, S, S, S), float('nan'))
    c = coords.copy()
    c[:, 1:] //= ts
    out[c[:, 0], :, c[:, 1], c[:, 2], c[:, 3]] = torch.as_tensor(rows)
    return out


@pytest.mark.parametrize('ks,stride,pad', [(2, 2, 0), (3, 1, 1), (3, 2, 1)])
def test_max_and_avg_equal_dense_pooling_and_autograd_on_full_grids(ks, stride, pad):
    B, C, S = 2, 3, 8
    dense, coords, feats = _dense_case(ks * 10 + stride, B, C, S)
    om = me_cpu.CoordinateManager(coords)
    ts_out = om.stride(1, stride) if stride > 1 else 1
    nbr = _nbr(om, 1, ts_out, ks)
    co = om.coords[ts_out]
    So = (S + 2 * pad - ks) // stride + 1
    gd = torch.randn(B, C, So, So, So, generator=torch.Generator().manual_seed(3))
    g_rows = gd[co[:, 0], :, co[:, 1] // ts_out, co[:, 2] // ts_out, co[:, 3] // ts_out].numpy()
    for mode in (P.MAX, P.AVG):
        d = dense.clone().requires_grad_(True)
        if mode == P.MAX:
            ref = F.max_pool3d(d, ks, stride, pad)
        else:
            ref = F.avg_pool3d(d, ks, stride, pad, count_include_pad=False)
        (ref * gd).sum().backward()
        out, cnt, win = P.pool_fwd(feats.numpy(), nbr, mode)
        got = _to_dense(out, co, ts_out, B, C, So)
        gin = P.pool_bwd(g_rows, nbr, mode, cnt, win, len(coords))
        ggot = _to_dense(gin, coords, 1, B, C, S)
        if mode == P.MAX:
            assert torch.equal(got, ref.detach())
        else:
            torch.testing.assert_close(got, ref.detach(), rtol=2e-6, atol=0)
        torch.testing.assert_close(ggot, d.grad, rtol=1e-5, atol=1e-6)       # summation order differs


NAN, INF = float('nan'), float('inf')


def _one(vals, present=None):
    """one output over K = len(vals) offsets, one channel; present[k] False drops offset k"""
    K = len(vals)
    x = np.asarray(vals, np.float32)[:, None]
    nbr = np.arange(K)[:, None].copy()
    if present is not None:
        nbr[~np.asarray(present), 0] = -1
    return x, nbr


@pytest.mark.parametrize('vals,present,value,winner', [
    ([1, 3, 3, 2], None, 3.0, 1),                       # tie: the lowest k
    ([1, NAN, 5, NAN], None, NAN, 1),                   # the first NaN
    ([NAN, INF], None, NAN, 0),
    ([INF, NAN], None, NAN, 1),
    ([-0.0, 0.0], None, -0.0, 0),                       # -0 == +0: the first
    ([0.0, -0.0], None, 0.0, 0),
    ([-INF, -INF], None, -INF, 0),
    ([-INF, -5], None, -5.0, 1),
    ([9, 2, 4], [False, True, True], 4.0, 2),           # absent offsets take no part
    ([7, 8], [False, False], 0.0, P.NO_WINNER),         # nothing present: 0, no winner
])
def test_max_rules_on_hand_built_windows(vals, present, value, winner):
    x, nbr = _one(vals, present)
    out, cnt, win = P.pool_fwd(x, nbr, P.MAX)
    assert _bits(out[0, 0]) == _bits(np.float32(value)) or (np.isnan(value) and np.isnan(out[0, 0]))
    assert win[0, 0] == winner
    gin = P.pool_bwd(np.array([[2.5]], np.float32), nbr, P.MAX, cnt, win, len(vals))
    exp = np.zeros((len(vals), 1), np.float32)
    if winner != P.NO_WINNER:
        exp[winner] = 2.5
    assert np.array_equal(gin, exp)


def test_sum_and_avg_rules_on_hand_built_windows():
    x, nbr = _one([1.0, -0.0, 2.0**-30, 3.0], [True, True, True, False])
    s, cnt, _ = P.pool_fwd(x, nbr, P.SUM)
    assert s[0, 0] == np.float32(1.0) + np.float32(2.0**-30) and cnt[0] == 3   # fp32 adds: 2^-30 is lost below 1
    a, _, _ = P.pool_fwd(x, nbr, P.AVG)
    assert a[0, 0] == np.float32(1.0) / np.float32(3)
    x, nbr = _one([-0.0], [True])
    s, _, _ = P.pool_fwd(x, nbr, P.SUM)
    assert _bits(s[0, 0]) == 0                                              # +0.0 + -0.0 = +0.0
    x, nbr = _one([5.0], [False])
    a, cnt, _ = P.pool_fwd(x, nbr, P.AVG)
    assert a[0, 0] == 0 and cnt[0] == 0
    gin = P.pool_bwd(np.array([[3.0]], np.float32), _one([1, 1, 1])[1], P.AVG, np.array([3], np.int32), None, 3)
    assert np.array_equal(gin[:, 0], np.full(3, np.float32(3.0) / np.float32(3.0)))


def test_global_rules():
    x = np.array([[1, NAN], [5, 2], [5, NAN], [-0.0, 7], [0.0, 7]], np.float32)
    batch = np.array([0, 0, 0, 2, 2])
    out, cnt, arg = P.global_fwd_exact(x, batch, 3, P.MAX)
    assert np.array_equal(arg, [[1, 0], [-1, -1], [3, 3]])
    assert out[0, 0] == 5 and np.isnan(out[0, 1]) and np.all(out[1] == -np.inf) and _bits(out[2, 0]) == 0x80000000
    s, cnt, _ = P.global_fwd_exact(x[:, :1], batch, 3, P.SUM)
    assert s[:, 0].tolist() == [11, 0, 0] and cnt.tolist() == [3, 0, 2]
    a, _, _ = P.global_fwd_exact(x[:, :1], batch, 3, P.AVG)
    assert a[0, 0] == np.float32(11 / 3) and np.isnan(a[1, 0])
    g = np.array([[3, 1], [4, 4], [6, 6]], np.float32)
    assert np.array_equal(P.global_bwd(g, batch, P.MAX, cnt, arg), [[0, 1], [3, 0], [0, 0], [6, 6], [0, 0]])
    assert np.array_equal(P.global_bwd(g, batch, P.AVG, cnt, arg)[:, 0], np.float32([1, 1, 1, 3, 3]))


# ------------------------------------------------------------------ mutated restatements must be caught
def test_mutants_are_caught():
    cl = synth.random_cloud(1200, 16, seed=9, batch=2)
    x = torch.randn(len(cl), 5, generator=torch.Generator().manual_seed(1))
    om = me_cpu.CoordinateManager(cl)
    xo = me_cpu.SparseTensor(x, coordinate_manager=om)
    ts2 = om.stride(1, 2)
    nbr = _nbr(om, 1, ts2, 2)
    ys = me_cpu.MinkowskiSumPooling(kernel_size=2, stride=2, dimension=3)(xo).F.numpy()
    ya = me_cpu.MinkowskiAvgPooling(kernel_size=2, stride=2, dimension=3)(xo).F.numpy()
    # a dropped last offset
    out, _, _ = P.pool_fwd(x.numpy(), nbr[:-1], P.SUM)
    assert not np.array_equal(_bits(out), _bits(ys))
    # average divided by the kernel volume instead of the count
    s, _, _ = P.pool_fwd(x.numpy(), nbr, P.SUM)
    assert not np.array_equal(_bits(s / np.float32(nbr.shape[0])), _bits(ya))
    # ties to the highest k (the offsets walked in reverse)
    xt, nt = _one([1, 3, 3, 2])
    _, _, w_rev = P.pool_fwd(xt, nt[::-1], P.MAX)
    assert nt.shape[0] - 1 - int(w_rev[0, 0]) != 1
    # and the dense check notices a dropped offset in max pooling too
    dense, coords, feats = _dense_case(5)
    om2 = me_cpu.CoordinateManager(coords)
    nb = _nbr(om2, 1, om2.stride(1, 2), 2)
    out, _, _ = P.pool_fwd(feats.numpy(), nb[:-1], P.MAX)
    got = _to_dense(out, om2.coords[2], 2, 2, 3, 4)
    assert not torch.equal(got, F.max_pool3d(dense, 2, 2))
