"""The fp64 references of tests/replay_ref.py (used by the GPU launch replay and the exact probes) against the CPU oracle
``oracle.me_cpu`` on small cases, and the split-row codec against its definition.  No GPU."""
import numpy as np
import pytest
import torch

from oracle import me_cpu
from openscene_b200 import synth
from tests import replay_ref as R


def _cloud(n=400, extent=9, seed=0):
    return synth.random_cloud(n, extent, seed=seed)


def _dense_map(maps, n_out):
    """me_cpu's [(in_rows, out_rows)] per offset -> output-stationary [K, n_out] (-1 = absent)"""
    nbr = torch.full((len(maps), n_out), -1, dtype=torch.int64)
    for k, (ii, oo) in enumerate(maps):
        nbr[k, oo] = ii
    return nbr


@pytest.mark.parametrize('ks,stride', [(3, 1), (2, 2), (1, 1)])
def test_conv_reference_matches_oracle(ks, stride):
    c = _cloud()
    om = me_cpu.CoordinateManager(c)
    ts_out = om.stride(1, stride) if stride > 1 else 1
    n_in, n_out = len(om.coords[1]), len(om.coords[ts_out])
    g = torch.Generator().manual_seed(ks)
    x = torch.randn(n_in, 40, generator=g, dtype=torch.float64)
    w = torch.randn(ks ** 3, 40, 24, generator=g, dtype=torch.float64)
    maps = om.kernel_map(1, ts_out, ks)
    ref = me_cpu._conv_apply(x, maps, w, n_out)
    nbr = None if ks == 1 else _dense_map(maps, n_out)
    y, a = R.conv(x, nbr, n_out, w)
    assert torch.allclose(y, ref, rtol=1e-12, atol=1e-12)
    ya, _ = R.conv(x.abs(), nbr, n_out, w.abs(), want_abs=False)
    assert torch.allclose(a, ya, rtol=1e-12, atol=1e-12)
    # epilogue: scale / shift / residual / ReLU and the abs scale
    s, b, r = torch.randn(24, generator=g), torch.randn(24, generator=g), torch.randn(n_out, 24, generator=g, dtype=torch.float64)
    ye, ae = R.epilogue(y, a, s, b, r, relu=True)
    assert torch.equal(ye, torch.relu(y * s.double() + b.double() + r))
    assert torch.equal(ae, a * s.double().abs() + b.double().abs() + r.abs())


def test_transposed_reference_matches_oracle():
    c = _cloud(seed=1)
    om = me_cpu.CoordinateManager(c)
    om.stride(1, 2)
    n_f, n_c = len(om.coords[1]), len(om.coords[2])
    g = torch.Generator().manual_seed(2)
    x = torch.randn(n_c, 32, generator=g, dtype=torch.float64)
    w = torch.randn(8, 32, 16, generator=g, dtype=torch.float64)
    conv = me_cpu.MinkowskiConvolutionTranspose(32, 16, kernel_size=2, stride=2, dimension=3).double()
    conv.kernel.data = w
    ref =conv(me_cpu.SparseTensor(x, coordinate_manager=om, tensor_stride=2)).F
    down = _dense_map(om.kernel_map(1, 2, 2), n_c)                 # child row of parent o through offset k
    y, _ = R.convtr(x, down, w, n_f)
    assert torch.allclose(y, ref, rtol=1e-12, atol=1e-12)
    # the same through the transposed map as an ordinary convolution
    y2, _ = R.conv(x, R.transpose_map(down, n_f), n_f, w)
    assert torch.allclose(y2, ref, rtol=1e-12, atol=1e-12)
    with pytest.raises(AssertionError, match='exactly once'):
        R.convtr(x, torch.cat([down[:1], down[:1], down[2:]]), w, n_f)


def test_transpose_map_definition():
    g = torch.Generator().manual_seed(3)
    n_in, n_out, K = 50, 40, 4
    nbr = torch.full((K, n_out), -1, dtype=torch.int64)
    for k in range(K):
        o = torch.randperm(n_out, generator=g)[:25]
        nbr[k, o] = torch.randperm(n_in, generator=g)[:25]
    t = R.transpose_map(nbr, n_in)
    for k in range(K):
        for o in range(n_out):
            if nbr[k, o] >= 0:
                assert t[k, nbr[k, o]] == o
        assert int((t[k] >= 0).sum()) == int((nbr[k] >= 0).sum())
    assert torch.equal(R.transpose_map(t, n_out), nbr)


@pytest.mark.parametrize('step', [1, 2])
def test_stem_neighbour_search_matches_oracle(step):
    c = _cloud(300, 7, seed=4).astype(np.int64)
    c[:, 1:] *= step
    c = np.concatenate([c, c[:40] * np.array([0, 1, 1, 1]) + np.array([1, 0, 0, 0])])     # a second batch index
    om = me_cpu.CoordinateManager(c)
    om.coords[step] = c                                  # the set at tensor stride `step`: neighbours step cells apart
    ref = _dense_map(om.kernel_map(step, step, 5), len(c))
    assert int((ref >= 0).sum()) > 3 * len(c)
    assert torch.equal(R.neighbour_map(torch.from_numpy(c).int(), 5, step), ref)


def test_wgrad_reference_matches_autograd():
    c = _cloud(seed=5)
    om = me_cpu.CoordinateManager(c)
    n = len(c)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(n, 32, generator=g, dtype=torch.float64)
    go = torch.randn(n, 16, generator=g, dtype=torch.float64)
    w = torch.randn(27, 32, 16, dtype=torch.float64, requires_grad=True)
    maps = om.kernel_map(1, 1, 3)
    (me_cpu._conv_apply(x, maps, w, n) * go).sum().backward()
    gw, a = R.wgrad(x, _dense_map(maps, n), go, 27)
    assert torch.allclose(gw, w.grad, rtol=1e-12, atol=1e-12)
    ga, _ = R.wgrad(x.abs(), _dense_map(maps, n), go.abs(), 27)
    assert torch.allclose(a, ga, rtol=1e-12, atol=1e-12)
    wi = torch.randn(1, 32, 16, dtype=torch.float64, requires_grad=True)
    ((x @ wi[0]) * go).sum().backward()
    assert torch.allclose(R.wgrad(x, None, go, 1)[0], wi.grad, rtol=1e-12, atol=1e-12)


def test_split_codec_matches_definition():
    g = torch.Generator().manual_seed(7)
    v = torch.randn(9, 64, generator=g) * torch.logspace(-20, 20, 64)
    raw = R.split_of(v)
    assert raw.dtype == torch.uint8 and raw.shape == (9, 256)
    # byte layout: per 32-channel block, 32 bf16 hi then 32 bf16 lo (little endian)
    hi = v.bfloat16()
    lo = (v - hi.float()).bfloat16()
    hb, lb = hi.view(torch.int16).numpy().astype('<i2'), lo.view(torch.int16).numpy().astype('<i2')
    for blk in range(2):
        line = raw[:, blk * 128:(blk + 1) * 128].numpy()
        assert (line[:, :64].copy().view('<i2') == hb[:, blk * 32:(blk + 1) * 32]).all()
        assert (line[:, 64:].copy().view('<i2') == lb[:, blk * 32:(blk + 1) * 32]).all()
    d = R.split_decode(raw, 64)
    assert torch.equal(d, hi.double() + lo.double())
    assert float(((d - v.double()).abs() / v.double().abs()).max()) <= 2.0 ** -17
    h2, l2 = R.split_halves(raw, 64)
    assert torch.equal(R.split_encode(h2, l2), raw)


def test_bounds_follow_the_plan():
    # osb_conv_wgrad_tc's row ranges: a partial last range and n_rs > 1 where the plan splits
    n_rs, rpr = R.wgrad_plan(10000, 1, 32, 32)
    assert n_rs > 1 and (n_rs - 1) * rpr < 10000 < n_rs * rpr and rpr % 128 == 0
    assert R.wgrad_plan(100, 27, 256, 256) == (1, 128)
    assert R.c_forward(27, 96) < R.c_forward(27, 384)
    assert 0.5 < R.c_forward(1, 32) < 2
    assert R.worst(torch.ones(3), torch.ones(3, dtype=torch.float64), torch.ones(3, dtype=torch.float64), 1.0) == 0.0
