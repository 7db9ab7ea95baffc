"""The CUDA-core bound, depths, dispatch restatement and probe operands of tests/replay_ref.py, checked without a GPU.

fp32 FMA chains are simulated in numpy (an fp32 product is exact in fp64, the sum is rounded once to fp32) in several orders,
including per-chunk partials followed by atomic adds in shuffled order, the way k_conv_wgrad_f32 and k_conv_wgrad_thin
accumulate; each must stay inside (depth + 3) 2^-24 A.  Negative controls alter a result the way a faulty kernel would (a
dropped offset, a dropped last row of a 4096-row chunk, a transposed weight, a missing last channel) and must break the
bound or the exact comparison."""
import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests import replay_ref as R


def _fma_chain(a, b, acc=None):
    """a, b float32 [T, m]: m independent fp32 FMA chains of T steps, as a CUDA thread runs them"""
    acc = np.zeros(a.shape[1], np.float32) if acc is None else acc
    for t in range(a.shape[0]):
        acc = (a[t].astype(np.float64) * b[t].astype(np.float64) + acc.astype(np.float64)).astype(np.float32)
    return acc


def _atomic_sum(partials, rng):
    """float atomic adds of per-block partials [P, m] into zero, each element in its own random order"""
    out = np.zeros(partials.shape[1], np.float32)
    order = np.argsort(rng.rand(*partials.shape), axis=0)
    for p in range(partials.shape[0]):
        out = (out + np.take_along_axis(partials, order[p:p + 1], 0)[0]).astype(np.float32)
    return out


def _terms(T, m, rng, spread=8):
    a = (rng.randn(T, m) * 2.0 ** rng.randint(-spread, spread + 1, (T, 1))).astype(np.float32)
    b = (rng.randn(T, m) * 2.0 ** rng.randint(-2, 3, (T, m))).astype(np.float32)
    ref = (a.astype(np.float64) * b.astype(np.float64)).sum(0)
    A = np.abs(a.astype(np.float64) * b.astype(np.float64)).sum(0)
    return a, b, torch.from_numpy(ref), torch.from_numpy(A)


def _fraction(y, ref, A, depth):
    c = R.c_fma(depth)
    return R.worst(torch.from_numpy(np.asarray(y)), ref, A, c) / c


@pytest.mark.parametrize('order', ['natural', 'reversed', 'shuffled', 'by_magnitude'])
def test_forward_chain_stays_in_bound_in_any_order(order):
    rng = np.random.RandomState(1)
    K, cin = 125, 3
    a, b, ref, A = _terms(K * cin, 512, rng)
    if order == 'reversed':
        a, b = a[::-1], b[::-1]
    elif order == 'shuffled':
        p = rng.permutation(K * cin)
        a, b = a[p], b[p]
    elif order == 'by_magnitude':                          # largest first: the worst case for absorbing the small terms
        p = np.argsort(-np.abs(a[:, 0]))
        a, b = a[p], b[p]
    y = _fma_chain(np.ascontiguousarray(a), np.ascontiguousarray(b))
    fr = _fraction(y, ref, A, R.f32_fwd_depth(K, cin))
    assert 0 < fr <= 1.0, fr


def test_generic_wgrad_chunks_and_shuffled_atomics_stay_in_bound():
    """k_conv_wgrad_f32: a 4096-row chunk per block, then ceil(n / 4096) atomic adds in any order"""
    rng = np.random.RandomState(2)
    n, m = 3 * R.WG_ROWS + 1, 48
    a, b, ref, A = _terms(n, m, rng)
    chunks = [_fma_chain(a[s:s + R.WG_ROWS], b[s:s + R.WG_ROWS]) for s in range(0, n, R.WG_ROWS)]
    y = _atomic_sum(np.stack(chunks), rng)
    assert len(chunks) == 4
    fr = _fraction(y, ref, A, R.f32_wgrad_depth('wgrad_generic', n))
    assert 0 < fr <= 1.0, fr


@pytest.mark.parametrize('n', [129, 67585])
def test_thin_wgrad_grid_stride_and_atomics_stay_in_bound(n):
    """k_conv_wgrad_thin: block b walks chunks b, b + grid, ... of 128 rows in one register, then one atomic add per block"""
    rng = np.random.RandomState(3)
    m = 16
    a, b, ref, A = _terms(n, m, rng)
    grid = R.thin_wgrad_grid(n)
    n_chunks = -(-n // R.THIN_WG_ROWS)
    pad = n_chunks * R.THIN_WG_ROWS - n
    ap, bp = np.concatenate([a, np.zeros((pad, m), np.float32)]), np.concatenate([b, np.zeros((pad, m), np.float32)])
    ap, bp = ap.reshape(n_chunks, R.THIN_WG_ROWS, m), bp.reshape(n_chunks, R.THIN_WG_ROWS, m)
    partials = []
    for blk in range(grid):
        acc = np.zeros(m, np.float32)
        for ch in range(blk, n_chunks, grid):
            acc = _fma_chain(ap[ch], bp[ch], acc)
        partials.append(acc)
    y = _atomic_sum(np.stack(partials), rng)
    fr = _fraction(y, ref, A, R.f32_wgrad_depth('wgrad_thin', n))
    assert 0 < fr <= 1.0, fr


def test_depths_follow_the_launch_plans():
    assert R.f32_fwd_depth(125, 3) == 375
    assert R.f32_wgrad_depth('wgrad_generic', 4096) == 4097 and R.f32_wgrad_depth('wgrad_generic', 4097) == 4098
    assert R.f32_wgrad_depth('wgrad_generic', 15) == 16
    # the thin wgrad's grid-stride loop starts above 528 x 128 rows
    assert R.thin_wgrad_grid(67584) == 528 and R.f32_wgrad_depth('wgrad_thin', 67584) == 128 + 528
    assert R.f32_wgrad_depth('wgrad_thin', 67585) == 256 + 528
    assert R.f32_wgrad_depth('wgrad_thin', 1) == 129
    # first order: depth 2^-24 stays far below 1 at the 197k-voxel scene
    assert R.f32_wgrad_depth('wgrad_generic', 197382) * 2.0 ** -24 < 2.0 ** -11
    assert R.f32_fwd_depth(343, 255) * 2.0 ** -24 < 2.0 ** -7


def test_dispatch_restatement():
    D = R.f32_dispatch
    assert D('fwd', 3, 32, 125, True) == 'fwd_thin'
    assert D('fwd', 3, 32, 256, True) == 'fwd_thin' and D('fwd', 3, 32, 257, True) == 'fwd_generic'   # 96 KiB of weights
    assert D('fwd', 1, 32, 768, True) == 'fwd_thin' and D('fwd', 1, 32, 769, True) == 'fwd_generic'
    assert D('fwd', 4, 32, 192, True) == 'fwd_thin' and D('fwd', 4, 32, 193, True) == 'fwd_generic'
    assert D('fwd', 3, 32, 27, True, ld_in=6) == 'fwd_generic'
    assert D('fwd', 3, 32, 27, True, transpose_w=True) == 'fwd_generic'
    assert D('fwd', 3, 32, 1, False) == 'fwd_generic'
    assert D('fwd', 5, 32, 27, True) == 'fwd_generic' and D('fwd', 3, 31, 27, True) == 'fwd_generic'
    assert D('wgrad', 3, 32, 128, True) == 'wgrad_thin' and D('wgrad', 3, 32, 129, True) == 'wgrad_generic'
    assert D('wgrad', 5, 32, 27, True) == 'wgrad_generic' and D('wgrad', 3, 32, 1, False) == 'wgrad_generic'
    assert D('wgrad', 4, 33, 27, True) == 'wgrad_generic'


def test_dyadic_probes_are_exact_in_any_order():
    """on the probe grid every fp32 partial is exact: any chain order and any atomic order give the fp64 sum bit for bit"""
    rng = np.random.RandomState(4)
    g = torch.Generator().manual_seed(4)
    n, m = 2 * R.WG_ROWS + 5, 32
    a = R.probe_x((n, m), g).numpy()
    b = R.probe_w((n, m), g).numpy()
    ref = (a.astype(np.float64) * b.astype(np.float64)).sum(0)
    A = torch.from_numpy(np.abs(a.astype(np.float64) * b.astype(np.float64)).sum(0))
    assert R.exact_budget_bits(A, R.PROBE_GRID) < 24
    for perm in (np.arange(n), rng.permutation(n)):
        parts = [_fma_chain(a[perm][s:s + R.WG_ROWS], b[perm][s:s + R.WG_ROWS]) for s in range(0, n, R.WG_ROWS)]
        assert np.array_equal(_atomic_sum(np.stack(parts), rng).astype(np.float64), ref)
    # the largest probes of the GPU tests stay inside the 2^24 budget by construction
    worst_fwd = 343 * 255 * 2 * 2.0 ** -3 * 3 * 2.0 ** -4
    worst_wgrad = 197382 * 2 * 2.0 ** -3 * 3 * 2.0 ** -4
    assert max(worst_fwd, worst_wgrad) / R.PROBE_GRID < 2.0 ** 21


# ------------------------------------------------------------------ negative controls
def _case(seed=5, n=300, cin=5, cout=5, K=27):
    c = torch.from_numpy(synth.random_cloud(n, 8, seed=seed)).int()
    nbr = R.neighbour_map(c, 3, 1)
    return c, nbr, len(c)


def _f32_conv(x, nbr, n_out, w):
    """what a correct kernel returns, to within the bound: the fp64 sum rounded to fp32"""
    return R.conv(x.double(), nbr, n_out, w.double(), want_abs=False)[0].float()


@pytest.mark.parametrize('control', ['dropped_offset', 'transposed_weight', 'missing_last_channel'])
def test_forward_negative_controls_break_the_bound_and_the_probe(control):
    c, nbr, n = _case()
    g = torch.Generator().manual_seed(6)
    cin = cout = 5
    for mode in ('bound', 'exact'):
        if mode == 'exact':
            x, w = R.probe_x((n, cin), g), R.probe_w((27, cin, cout), g)
        else:
            x, w = R.binade_rows(n, cin, 8, g), R.binade_rows(27 * cin, cout, 2, g).view(27, cin, cout)
        ref, A = R.conv(x.double(), nbr, n, w.double())
        good = _f32_conv(x, nbr, n, w)
        depth = R.f32_fwd_depth(27, cin)
        assert R.worst(good, ref, A, R.c_fma(depth)) <= R.c_fma(depth)
        if control == 'dropped_offset':
            m = nbr.clone()
            m[13] = -1                                           # the centre offset: every row has it
            bad = _f32_conv(x, m, n, w)
        elif control == 'transposed_weight':
            bad = _f32_conv(x, nbr, n, w.transpose(1, 2).contiguous())
        else:
            xm = x.clone()
            xm[:, -1] = 0
            bad = _f32_conv(xm, nbr, n, w)
        if mode == 'exact':
            assert torch.equal(good.double(), ref) and not torch.equal(bad.double(), ref)
        else:
            assert R.worst(bad, ref, A, R.c_fma(depth)) > 100 * R.c_fma(depth)


def test_wgrad_dropped_last_chunk_row_hides_in_the_bound_but_not_the_probe():
    """a weight gradient that drops the last row of the first 4096-row chunk: within a depth-linear bound at this size,
    caught by the exact probe"""
    g = torch.Generator().manual_seed(7)
    n, cin, cout = 3 * R.WG_ROWS + 1, 3, 4
    keep = torch.ones(n, dtype=torch.bool)
    keep[R.WG_ROWS - 1] = False
    for mode in ('bound', 'exact'):
        if mode == 'exact':
            x, go = R.probe_x((n, cin), g), R.probe_w((n, cout), g)
            x[R.WG_ROWS - 1] = 2.0 ** -3                          # the dropped rows carry something
            go[R.WG_ROWS - 1] = 2.0 ** -4
        else:
            x, go = torch.rand((n, cin), generator=g) + 1, torch.rand((n, cout), generator=g) + 1
        ref, A = R.wgrad(x.double(), None, go.double(), 1)
        bad = R.wgrad(x[keep].double(), None, go[keep].double(), 1)[0].float()
        if mode == 'exact':
            assert R.exact_budget_bits(A, R.PROBE_GRID) < 24
            assert not torch.equal(bad.double(), ref)
        else:
            depth = R.f32_wgrad_depth('wgrad_generic', n)
            assert R.worst(bad, ref, A, R.c_fma(depth)) <= R.c_fma(depth)        # this is why the probes exist
