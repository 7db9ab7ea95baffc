"""The cross-entropy head kernels (osb_ce_head_fwd / osb_ce_head_bwd) through the C ABI against fp64 torch, computed on exactly
the values the split rows hold.

Bounds: loss within 2^-20 relative; pred equal to the fp64 argmax wherever the row's top-two gap exceeds 2^-18 max|z|; two runs
bit-identical.  dx and dW: the kernels form z in fp32 (k ascending) and read lse as fp32, so softmax(z) carries the relative
error exp(dz - dlse) - 1 with |dz - dlse| <= 2^-18 (max_c sum_k |x_k w_kc| + |lse|) (fp32 dot of <= 384 terms plus the
rounding of lse).  At |z| ~ 1e3 that is ~4e-3 absolute in the exponent, far above the operand rounding the flat bounds cover,
so each carries that term as well:
  dx_rk: 2^-17 |dx_rk| + 2^-22 sum_c |d_rc| |w_kc| + eps_r sum_c |p_rc s| |w_kc|
  dW_kc: (rows per split + 5) 2^-24 sum_r |x_rk| |d_rc| + sum_r |x_rk| eps_r |p_rc s|   (tests/norm_ref.py ce_dw_bound;
         eps_r = 2^-18 (zabs_r + |lse_r|), s = g / n_valid)
For logits of order one the extra terms are ~2^-15 of the flat ones."""
import pytest
import torch

from openscene_b200 import _cabi as C
from tests import norm_ref as NR

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _joined(rows, c):
    out = torch.empty((rows.shape[0], c), dtype=torch.float32, device=DEV)
    C.call('osb_split_to_f32', C.ptr(rows), rows.shape[0], c, C.ptr(out), C.stream_ptr())
    return out


def _case(n, cin, c, seed, scale=1.0, i64=True, ignore=255, frac_ignored=0.15):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, generator=g)
    w = torch.randn(cin, c, generator=g) / cin ** 0.5 * scale
    perm = torch.randperm(n, generator=g).to(torch.int32)
    lab = torch.randint(0, c, (n,), generator=g)
    lab[torch.rand(n, generator=g) < frac_ignored] = ignore
    lab = lab.to(torch.int64 if i64 else torch.int32)
    return _split(x.to(DEV)), w.to(DEV), perm.to(DEV), lab.to(DEV)


def _run(xs, n, cin, w, c, perm, lab, ignore, g=1.0):
    ws_b = C.lib().osb_ce_head_workspace_bytes(n, cin, c)
    ws = torch.empty(ws_b, dtype=torch.uint8, device=DEV)
    lse = torch.empty(n, device=DEV)
    pred = torch.empty(n, dtype=torch.int64, device=DEV)
    loss = torch.empty(1, device=DEV)
    nv = torch.empty(1, dtype=torch.int64, device=DEV)
    i64 = 1 if lab.dtype == torch.int64 else 0
    C.call('osb_ce_head_fwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(perm), C.ptr(lab), i64, ignore, C.ptr(lse), C.ptr(pred),
           C.ptr(loss), C.ptr(nv), C.ptr(ws), ws_b, C.stream_ptr())
    gt = torch.full((1,), g, device=DEV)
    dx = torch.empty((n, 4 * cin), dtype=torch.uint8, device=DEV)
    dw = torch.empty((cin, c), device=DEV)
    C.call('osb_ce_head_bwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(perm), C.ptr(lab), i64, ignore, C.ptr(lse), C.ptr(gt),
           C.ptr(nv), C.ptr(dx), C.ptr(dw), C.ptr(ws), ws_b, C.stream_ptr())
    torch.cuda.synchronize()
    return lse, pred, loss, nv, dx, dw


def _reference(xs, cin, w, perm, lab, ignore, g=1.0):
    """fp64 autograd on the joined split values, rows in internal order (labels gathered through perm)"""
    x = _joined(xs, cin).double().requires_grad_()
    w64 = w.double().requires_grad_()
    lab_int = lab.long()[perm.long()]
    z = x @ w64
    loss = torch.nn.functional.cross_entropy(z, lab_int, ignore_index=ignore)
    (loss * g).backward()
    return z.detach(), loss.detach(), x.grad, w64.grad, lab_int


def _check(xs, n, cin, w, c, perm, lab, ignore, g=1.0):
    lse, pred, loss, nv, dx, dw = _run(xs, n, cin, w, c, perm, lab, ignore, g)
    z, l64, dx64, dw64, lab_int = _reference(xs, cin, w, perm, lab, ignore, g)
    labelled = lab_int != ignore
    assert int(nv) == int(labelled.sum())
    lse64 = torch.logsumexp(z, 1)
    assert torch.allclose(lse.double(), lse64, rtol=2 ** -20, atol=2 ** -20 * float(lse64.abs().max()))
    if int(nv) == 0:
        assert torch.isnan(loss).all()
        assert torch.count_nonzero(dx) == 0 and torch.count_nonzero(dw) == 0
        return
    assert abs(float(loss) - float(l64)) <= 2 ** -20 * abs(float(l64)), (float(loss), float(l64))
    # pred in caller order; the fp64 argmax wherever the top-two gap is resolvable
    pred_int = pred[perm.long()]
    top2 = z.topk(min(2, c), 1).values
    gap = top2[:, 0] - top2[:, 1] if c > 1 else torch.full((n,), float('inf'), dtype=torch.float64, device=DEV)
    sure = gap > 2 ** -18 * z.abs().max(1).values
    assert torch.equal(pred_int[sure], z.argmax(1)[sure])
    # gradients
    x64 = _joined(xs, cin).double()
    w64 = w.double()
    s = g / int(nv)
    p = torch.softmax(z, 1) * s * labelled[:, None]
    d64 = p - torch.nn.functional.one_hot(lab_int.clamp(0, c - 1), c).double() * s * labelled[:, None]
    zabs = (x64.abs() @ w64.abs()).max(1).values
    eps = 2 ** -18 * (zabs + lse64.abs())
    dxf = _joined(dx, cin).double()
    bound_dx = 2 ** -17 * dx64.abs() + 2 ** -22 * (d64.abs() @ w64.abs().t()) + eps[:, None] * (p.abs() @ w64.abs().t())
    assert bool(((dxf - dx64).abs() <= bound_dx + 1e-30).all()), float(((dxf - dx64).abs() - bound_dx).max())
    bound_dw = NR.ce_dw_bound(x64, dict(d=d64, p=p, eps=eps), n)
    assert bool(((dw.double() - dw64).abs() <= bound_dw).all()), float(((dw.double() - dw64).abs() - bound_dw).max())


SHAPES = [(32, 1), (96, 20), (96, 21), (128, 16), (96, 160), (384, 160)]


@pytest.mark.parametrize('n', [1, 37, 70001])
@pytest.mark.parametrize('cin,c', SHAPES)
@pytest.mark.parametrize('i64', [True, False])
def test_against_fp64(n, cin, c, i64):
    xs, w, perm, lab = _case(n, cin, c, seed=n + cin + c, i64=i64)
    _check(xs, n, cin, w, c, perm, lab, 255, g=0.75)


@pytest.mark.parametrize('cin,c', [(96, 20), (384, 160)])
def test_large_logits(cin, c):
    """|z| ~ 1e3: log-sum-exp stays finite and exact to the bounds"""
    xs, w, perm, lab = _case(5000, cin, c, seed=11, scale=1000.0)
    lse, *_ = _run(xs, 5000, cin, w, c, perm, lab, 255)
    assert torch.isfinite(lse).all() and float(lse.abs().max()) > 300
    _check(xs, 5000, cin, w, c, perm, lab, 255)


def test_exact_ties_take_the_first_maximum():
    n, cin, c = 300, 96, 21
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, cin, generator=g)
    w = torch.randn(cin, c, generator=g) / 10
    tie = torch.randint(0, c, (n,), generator=g)
    w[:, 7] = w[:, 3]                                    # classes 3 and 7 (and 19 / 20) always tie
    w[:, 20] = w[:, 19]
    x[:100] = 0.0                                        # all-zero rows: every class ties, pred = 0
    perm = torch.randperm(n, generator=g).to(torch.int32).to(DEV)
    xs = _split(x.to(DEV))
    lab = tie.to(DEV)
    _, pred, *_ = _run(xs, n, cin, w.to(DEV), c, perm, lab, -100)
    z = _joined(xs, cin).double() @ w.double().to(DEV)
    pred_int = pred[perm.long()]
    assert torch.equal(pred_int, z.argmax(1))           # torch's argmax takes the first maximum as well
    assert bool((pred_int[:100] == 0).all())
    assert not bool(((pred_int == 7) | (pred_int == 20)).any())


@pytest.mark.parametrize('i64', [True, False])
def test_all_ignored(i64):
    n, cin, c = 1000, 96, 20
    xs, w, perm, lab = _case(n, cin, c, seed=5, i64=i64, frac_ignored=1.0)
    _check(xs, n, cin, w, c, perm, lab, 255)


@pytest.mark.parametrize('cin,c', [(96, 20), (384, 160)])
def test_two_runs_identical(cin, c):
    n = 70001
    xs, w, perm, lab = _case(n, cin, c, seed=9)
    a = _run(xs, n, cin, w, c, perm, lab, 255)
    b = _run(xs, n, cin, w, c, perm, lab, 255)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
