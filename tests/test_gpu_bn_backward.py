"""The training kernels of csrc/bn_train.cu through the C ABI: ``osb_bn_batch_stats_save`` (batch mean / invstd kept),
``osb_bn_apply_split_out`` (normalised rows next to the raw ones) and the backward of relu(BN(z) + r),
``osb_bn_backward_reduce`` / ``osb_bn_backward_apply``, against fp64 autograd of ``F.batch_norm(training=True)`` in all three
residual forms, with per-channel means up to 10^3 sigma."""
import pytest
import torch
import torch.nn.functional as F

from openscene_b200 import _cabi as C
from tests import norm_ref as NR

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _to_split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _joined(rows, c):
    out = torch.empty((rows.shape[0], c), dtype=torch.float32, device=DEV)
    C.call('osb_split_to_f32', C.ptr(rows), rows.shape[0], c, C.ptr(out), C.stream_ptr())
    return out


@pytest.mark.parametrize('relu', [1, 0])
@pytest.mark.parametrize('form', ['none', 'identity', 'normalised'])
@pytest.mark.parametrize('n,c', [(3, 32), (4099, 96), (197383, 64)])
def test_bn_backward_kernels_match_fp64_autograd(n, c, form, relu):
    """relu=0: no activation after the add, so the backward gets y_split = NULL (no mask).  Channel 0 has weight 0 (scale and
    shift carry no trace of the statistics there, which is why the forward saves mean / invstd)."""
    g_ = torch.Generator(device=DEV).manual_seed(n + c)
    sigma = torch.exp(4 * torch.rand(c, device=DEV, generator=g_) - 2)
    mean = sigma * (2000 * torch.rand(c, device=DEV, generator=g_) - 1000)
    z_rows = _to_split(mean + sigma * torch.randn(n, c, device=DEV, generator=g_))
    r_rows = _to_split(3 * torch.randn(n, c, device=DEV, generator=g_) + 1)
    g_rows = _to_split(torch.randn(n, c, device=DEV, generator=g_))
    z, r, gin = (_joined(t, c).double() for t in (z_rows, r_rows, g_rows))
    w = (0.5 + torch.rand(c, device=DEV, generator=g_))
    w[0] = 0.0
    b = torch.rand(c, device=DEV, generator=g_) - 0.5
    rm, rv, nbt = torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    scale, shift, mu, istd = (torch.empty(c, device=DEV) for _ in range(4))
    ws_bytes = C.lib().osb_bn_stats_workspace_bytes(n, c)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    C.call('osb_bn_batch_stats_save', z_rows.data_ptr(), n, c, w.data_ptr(), b.data_ptr(), 1e-5, 0.1, rm.data_ptr(), rv.data_ptr(),
           nbt.data_ptr(), scale.data_ptr(), shift.data_ptr(), mu.data_ptr(), istd.data_ptr(), ws.data_ptr(), ws_bytes,
           C.stream_ptr())
    rsc = rsh = None
    if form == 'normalised':            # the residual is a raw downsample output normalised with its own scale / shift
        rsc, rsh = 0.5 + torch.rand(c, device=DEV, generator=g_), torch.rand(c, device=DEV, generator=g_)
    y_rows = torch.empty_like(z_rows)
    C.call('osb_bn_apply_split_out', z_rows.data_ptr(), y_rows.data_ptr(), n, c, scale.data_ptr(), shift.data_ptr(),
           None if form == 'none' else r_rows.data_ptr(), C.ptr(rsc), C.ptr(rsh), relu, C.stream_ptr())
    # fp64 autograd of relu(batch_norm(z) + r)
    zz, ww, bb = z.clone().requires_grad_(), w.double().requires_grad_(), b.double().requires_grad_()
    t = F.batch_norm(zz, None, None, ww, bb, training=True, eps=1e-5)
    rr = torch.zeros_like(t) if form == 'none' else (r if form == 'identity' else r * rsc.double() + rsh.double())
    yy = torch.relu(t + rr) if relu else t + rr
    yy.backward(gin)
    # the forward: mean / invstd saved, y out of place, z untouched
    assert float(((mu.double() - z.mean(0)).abs() / sigma.double()).max()) < 1e-4
    var = z.var(0, unbiased=False)
    assert float((istd.double() * torch.sqrt(var + 1e-5) - 1).abs().max()) < 1e-5
    assert torch.equal(_joined(z_rows, c).double(), z)
    # y on the kernel's own fp32 scale / shift, with the bound of tests/test_gpu_bn_batch_stats.py
    y = _joined(y_rows, c).double()
    t_k = z * scale.double() + shift.double()
    r_k = torch.zeros_like(t_k) if form == 'none' else (r if form == 'identity' else r * rsc.double() + rsh.double())
    y_ref = (t_k + r_k).clamp_min(0) if relu else t_k + r_k
    assert bool(((y - y_ref).abs() <= 2.0 ** -17 * y_ref.abs() + 2.0 ** -22 * (t_k.abs() + shift.double().abs() + r_k.abs())).all())
    # the backward, on the kernel's own forward output (its ReLU mask)
    sums = torch.empty(2 * c, device=DEV)
    dw, db = torch.empty(c, device=DEV), torch.empty(c, device=DEV)
    dz_rows, gp_rows = torch.empty_like(z_rows), torch.empty_like(z_rows)

    y_arg = y_rows.data_ptr() if relu else None

    def run():
        C.call('osb_bn_backward_reduce', y_arg, g_rows.data_ptr(), z_rows.data_ptr(), n, c, mu.data_ptr(), istd.data_ptr(),
               sums.data_ptr(), dw.data_ptr(), db.data_ptr(), 0, ws.data_ptr(), ws_bytes, C.stream_ptr())
        C.call('osb_bn_backward_apply', y_arg, g_rows.data_ptr(), z_rows.data_ptr(), n, c, mu.data_ptr(),
               istd.data_ptr(), w.data_ptr(), sums.data_ptr(), dz_rows.data_ptr(), gp_rows.data_ptr(), 0, C.stream_ptr())
        return [t.clone() for t in (dw, db, dz_rows, gp_rows)]
    first = run()
    # the reference's mask is its own y > 0; rows where the two forwards disagree on the sign are excluded from dz
    gp_ref = gin * (y > 0) if relu else gin
    xh = (z - z.mean(0)) * torch.rsqrt(var + 1e-5)
    dw_ref, db_ref = (gp_ref * xh).sum(0), gp_ref.sum(0)
    same = ((y > 0) == (yy.detach() > 0)).all(1) if relu else torch.ones(n, dtype=torch.bool, device=DEV)
    assert float(dw[0]) != 0.0 and float(_joined(dz_rows, c)[:, 0].abs().max()) == 0.0   # weight 0: dz 0
    # dweight / dbias per channel against the operands the launch read (the kernel's mask, saved mean / invstd):
    # tests/norm_ref.py's depth term plus one fp32 rounding
    bw = NR.bn_backward(y if relu else None, gin, z, mu, istd, w)
    rb0 = NR.reduce_bounds(bw)
    assert bool(((dw.double() - bw['t2']).abs() <= rb0['dweight']).all())
    assert bool(((db.double() - bw['t1']).abs() <= rb0['dbias']).all())
    dz_ref = ww.detach() * torch.rsqrt(var + 1e-5) * (gp_ref - db_ref / n - xh * dw_ref / n)
    dz = _joined(dz_rows, c).double()
    a = (ww.detach() * torch.rsqrt(var + 1e-5)).abs()
    # a split row holds dz to 2^-17; the fp32 evaluation rounds its operands (g', the sums / n, x^ from the fp32 mean) to 2^-24
    # plus the fp32 rounding of the saved mean: it shifts every x^ of a channel by d <= 2^-24 |mean| invstd, which moves
    # sum g' x^ / n by d sum g' / n and dz by weight invstd d (|sum g' x^ / n| + |x^ sum g' / n|) to first order
    d = 2.0 ** -23 * z.mean(0).abs() * torch.rsqrt(var + 1e-5)
    tol = (2.0 ** -17 * dz_ref.abs() + 2.0 ** -21 * a * (gp_ref.abs() + (db_ref / n).abs() + (xh * dw_ref / n).abs())
           + a * d * ((dw_ref / n).abs() + (xh * db_ref / n).abs()))
    ok = ((dz - dz_ref).abs() <= tol) | ~same.unsqueeze(1)
    assert bool(ok.all()), float(((dz - dz_ref).abs() / (tol + 1e-30))[same].max())
    assert n < 100 or float(same.double().mean()) > 0.999
    assert torch.equal(_joined(gp_rows, c).double()[same], gp_ref[same])
    # accumulate modes, and two runs bit-identical
    second = run()
    assert all(torch.equal(p, q) for p, q in zip(first, second))
    C.call('osb_bn_backward_reduce', y_arg, g_rows.data_ptr(), z_rows.data_ptr(), n, c, mu.data_ptr(), istd.data_ptr(),
           sums.data_ptr(), dw.data_ptr(), db.data_ptr(), 1, ws.data_ptr(), ws_bytes, C.stream_ptr())
    # accumulate: one fp32 rounding of prev + t (tests/norm_ref.py).  prev = fp32(t) here, so a double rounding
    # prev + fp32(t) = fp32(2 t) would not show; tests/test_gpu_bn_exact.py accumulates onto independent values
    rb = NR.reduce_bounds(bw, first[0], first[1])
    assert bool(((dw.double() - rb['dw_ref']).abs() <= rb['dweight']).all())
    assert bool(((db.double() - rb['db_ref']).abs() <= rb['dbias']).all())
    C.call('osb_bn_backward_apply', y_arg, g_rows.data_ptr(), z_rows.data_ptr(), n, c, mu.data_ptr(),
           istd.data_ptr(), w.data_ptr(), sums.data_ptr(), dz_rows.data_ptr(), gp_rows.data_ptr(), 1, C.stream_ptr())
    gp2 = _joined(gp_rows, c).double()
    assert float((gp2 - 2 * gp_ref)[same].abs().max()) <= 2.0 ** -16 * float(gp_ref.abs().max())
