"""The cosine distillation head kernels (osb_cos_head_fwd / osb_cos_head_bwd) through the C ABI against fp64 torch, computed on
exactly the values the kernels multiply: the split rows joined (x), the fp32 weights (W) and the fp16 targets widened (t).

Bounds, u = 2^-24, g_k = k u / (1 - k u), E = g_cin |X| |W| the error bound of the fp32 products f = x W:
  state  | |f|dev - |f| | <= dn1 = |E_r|_2,  |f.t dev - f.t| <= dft = sum_j E_rj |t_rj|  (the sums themselves are fp64);
         |t| to 1e-12 relative (fp64 sums of exact products)
  loss   <= sum_r (dft_r / (n1c n2c) + |cos_r| dn1_r / n1c) / m + u |loss|
  a, b   the fp64 (a, b) of the state rounded to fp32:
         da <= |a| (dn1 / n1c + u),  db <= |b| (3 dn1 / n1 + u) + g dft / (m n1c^2 n2c n1)
  dx_rk  = a P + b Q, P = t W^T (fp32, C terms), Q = x G (fp32, cin terms), G = W W^T (fp32, C terms):
         da |P| + |a| g_C (|t| |W|^T) + db |Q| + |b| (g_cin |x| |G| + |x| g_C (|W| |W|^T)) + u (|a P| + 2 |b Q|)
         + 2^-17 |dx| (the split store)
  dW_kj  = sum_r a_r x_rk t_rj (fp32 over the rows of one split, after one rounding of a t; splits merged in fp64)
         + sum_i H_ki W_ij (H = sum_r b_r x_rk x_ri the same way, the product with W in fp64):
         sum_r (da_r + g_{s+1} |a_r|) |x_rk| |t_rj| + sum_i |W_ij| sum_r (db_r + g_{s+1} |b_r|) |x_rk| |x_ri| + u |dW|,
         s = rows per split = ceil(m / min(ceil(m / 512), 64))
Every bound gets a factor 1.5 for the second-order terms dropped above.  Edge rows (tests/cos_ref.py's list): a zero output
row (x = 0), 0 < |f| < eps (x one small channel, so x W does not cancel), a zero target row (dx exactly 0) and, in a call of
its own, a NaN row (the loss is NaN)."""
import math

import pytest
import torch

from openscene_b200 import _cabi as C
from tests import cos_ref

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24


def _gam(k):
    return k * U / (1 - k * U)


def _split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _joined(rows, c):
    out = torch.empty((rows.shape[0], c), dtype=torch.float32, device=DEV)
    C.call('osb_split_to_f32', C.ptr(rows), rows.shape[0], c, C.ptr(out), C.stream_ptr())
    return out


def _case(m, cin, c, seed, edges=False):
    g = torch.Generator().manual_seed(seed)
    n = m + m // 2 + 7                                       # unsupervised rows too
    x = torch.randn(n, cin, generator=g)
    w = torch.randn(cin, c, generator=g) / cin ** 0.5
    rows = torch.randperm(n, generator=g)[:m].to(torch.int32)
    t = torch.randn(m, c, generator=g).half()
    if edges:
        r = rows.long()
        x[r[1]] = 0                                          # zero output row
        x[r[2]] = 0
        x[r[2], 5] = 1e-10                                   # 0 < |f| < eps, no cancellation
        t[3] = 0                                             # zero target row
    return _split(x.to(DEV)), w.to(DEV), rows.to(DEV), t.to(DEV)


def _run(xs, cin, w, c, rows, t, g=1.0):
    n, m = xs.shape[0], rows.shape[0]
    ws_b = C.lib().osb_cos_head_workspace_bytes(m, cin, c)
    ws = torch.empty(ws_b, dtype=torch.uint8, device=DEV)
    state = torch.empty((m, 3), dtype=torch.float64, device=DEV)
    loss = torch.empty(1, device=DEV)
    C.call('osb_cos_head_fwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(rows), m, C.ptr(t), C.ptr(state), C.ptr(loss), C.ptr(ws),
           ws_b, C.stream_ptr())
    gt = torch.full((1,), g, device=DEV)
    dx = torch.full((n, 4 * cin), 0x7f, dtype=torch.uint8, device=DEV)    # poisoned: every row must be written
    dw = torch.full((cin, c), float('nan'), device=DEV)
    C.call('osb_cos_head_bwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(rows), m, C.ptr(t), C.ptr(state), C.ptr(gt), C.ptr(dx),
           C.ptr(dw), C.ptr(ws), ws_b, C.stream_ptr())
    torch.cuda.synchronize()
    return state, loss, dx, dw


def _check(xs, cin, w, c, rows, t, g=1.0):
    state, loss, dx, dw = _run(xs, cin, w, c, rows, t, g)
    m = rows.shape[0]
    r = rows.long()
    X = _joined(xs, cin).double()[r]
    W, T = w.double(), t.double()
    F = X @ W
    n1, n2, ft = F.norm(dim=1), T.norm(dim=1), (F * T).sum(1)
    n1c, n2c = n1.clamp_min(cos_ref.EPS), n2.clamp_min(cos_ref.EPS)
    cos = ft / (n1c * n2c)
    loss_ref = (1 - cos).mean()
    E = _gam(cin) * (X.abs() @ W.abs())
    dn1 = E.norm(dim=1)
    dft = (E * T.abs()).sum(1)
    assert (state[:, 0] - n1).abs().le(1.5 * dn1 + 1e-12 * n1).all()
    assert (state[:, 1] - ft).abs().le(1.5 * dft + 1e-12 * (F * T).abs().sum(1)).all()
    assert (state[:, 2] - n2).abs().le(1e-12 * n2).all()
    lb = ((dft / (n1c * n2c) + cos.abs() * dn1 / n1c).sum() / m + U * loss_ref.abs()) * 1.5
    assert abs(float(loss) - float(loss_ref)) <= float(lb), (float(loss), float(loss_ref), float(lb))

    a, b = cos_ref.cos_ab(n1, ft, n2, m, g)
    n1s = n1.clamp_min(1e-300)
    da = a.abs() * (dn1 / n1c + U)
    db = torch.where(n1 > 0, b.abs() * (3 * dn1 / n1s + U) + g * dft / (m * n1c * n1c * n2c * n1s), torch.zeros_like(n1))
    P, Q = T @ W.t(), F @ W.t()
    G = W @ W.t()
    dxr = a[:, None] * P + b[:, None] * Q
    bx = (da[:, None] * P.abs() + a.abs()[:, None] * _gam(c) * (T.abs() @ W.abs().t())
          + db[:, None] * Q.abs() + b.abs()[:, None] * (_gam(cin) * (X.abs() @ G.abs()) + _gam(c) * (X.abs() @ (W.abs() @ W.abs().t())))
          + U * (a.abs()[:, None] * P.abs() + 2 * b.abs()[:, None] * Q.abs()) + 2.0 ** -17 * dxr.abs()) * 1.5
    dxd = _joined(dx, cin).double()
    assert ((dxd[r] - dxr).abs() <= bx).all(), float(((dxd[r] - dxr).abs() - bx).max())
    others = torch.ones(xs.shape[0], dtype=torch.bool, device=DEV)
    others[r] = False
    assert torch.equal(dx.view(xs.shape[0], -1)[others], torch.zeros_like(dx[others]))
    s = math.ceil(m / min(math.ceil(m / 512), 64))
    gs = _gam(s + 1)
    dwr = X.t() @ (a[:, None] * T) + (X.t() @ (b[:, None] * X)) @ W
    bw = ((X.abs().t() @ ((da + gs * a.abs())[:, None] * T.abs()))
          + (X.abs().t() @ ((db + gs * b.abs())[:, None] * X.abs())) @ W.abs() + U * dwr.abs()) * 1.5
    assert ((dw.double() - dwr).abs() <= bw).all(), float(((dw.double() - dwr).abs() - bw).max())
    return state, loss, dx, dw, dxr, r


@pytest.mark.parametrize('m,cin,c', [(1, 96, 768), (31, 384, 512), (20000, 96, 768), (20000, 384, 768), (20000, 96, 512),
                                     (160000, 96, 768)])
def test_against_fp64(m, cin, c):
    xs, w, rows, t = _case(m, cin, c, seed=m + cin + c)
    _check(xs, cin, w, c, rows, t, g=0.75)


def test_two_runs_are_bit_identical():
    xs, w, rows, t = _case(20000, 96, 768, seed=4)
    a = _run(xs, 96, w, 768, rows, t)
    b = _run(xs, 96, w, 768, rows, t)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.uint8) if u.dtype != torch.uint8 else u, v.view(torch.uint8) if v.dtype != torch.uint8 else v)


def test_edge_rows():
    m, cin, c = 300, 96, 768
    xs, w, rows, t = _case(m, cin, c, seed=9, edges=True)
    state, loss, dx, dw, dxr, r = _check(xs, cin, w, c, rows, t)
    assert float(state[1, 0]) == 0.0 and float(state[1, 1]) == 0.0       # zero output row: cos 0
    assert 0 < float(state[2, 0]) < cos_ref.EPS
    dxd = _joined(dx, cin).double()
    assert dxd[r[2]].abs().max() > 1e-2 / (m * cos_ref.EPS)              # gradients of order 1 / (M eps)
    assert torch.equal(dxd[r[3]], torch.zeros_like(dxd[r[3]]))           # zero target row: gradient exactly 0
    # the NaN rule: one NaN in a supervised row makes the loss NaN
    x = _joined(xs, cin)
    x[r[4], 7] = float('nan')
    _, loss, _, _ = _run(_split(x), cin, w, c, rows, t)
    assert math.isnan(float(loss))
