"""tests/cos_ref.py against torch.nn.CosineSimilarity in fp64 on the CPU: the restated loss and its autograd gradient are the
same bits, and the closed form the device head implements agrees with them (the edge rows exactly where it is exact).  The
bounds of ``cos_ref.head`` hold for an fp32 emulation of the head's documented arithmetic, on random and edge rows, and
mutated references (rows rolled by one, g = 1 in place of 0.75, W after one Adam step) fall outside them."""
import torch

from tests import cos_ref
from tests import replay_ref as R


def _torch(f, t):
    f = f.clone().requires_grad_(True)
    loss = (1 - torch.nn.CosineSimilarity(dim=1, eps=1e-8)(f, t)).mean()
    loss.backward()
    return loss.detach(), f.grad


def _restated(f, t):
    f = f.clone().requires_grad_(True)
    loss = cos_ref.cos_loss(f, t)
    loss.backward()
    return loss.detach(), f.grad


def test_restatement_is_bit_exact_on_random_rows():
    gen = torch.Generator().manual_seed(1)
    for c in (512, 768):
        f = torch.randn(257, c, generator=gen, dtype=torch.float64)
        t = torch.randn(257, c, generator=gen, dtype=torch.float64).half().double()
        lt, gt = _torch(f, t)
        lr, gr = _restated(f, t)
        assert torch.equal(lt, lr) and torch.equal(gt, gr)
        assert torch.allclose(cos_ref.cos_grad(f, t), gt, rtol=1e-12, atol=0)


def test_edge_rows():
    f, t = cos_ref.edge_rows(768)
    lt, gt = _torch(f, t)
    lr, gr = _restated(f, t)
    assert torch.isnan(lt) and torch.isnan(lr)
    assert torch.equal(torch.nan_to_num(gt, 7.0), torch.nan_to_num(gr, 7.0))
    fin, tin = f[:7], t[:7]                                    # without the NaN row
    lt, gt = _torch(fin, tin)
    lr, gr = _restated(fin, tin)
    assert torch.equal(lt, lr) and torch.equal(gt, gr)
    m = fin.shape[0]
    # zero output row: cos 0, gradient -t / (M eps |t|)
    assert torch.allclose(gt[1], -tin[1] / (m * 1e-8 * tin[1].norm()), rtol=1e-14, atol=0)
    # 0 < |f| < eps: gradients of order 1 / (M eps)
    assert gt[2].abs().max() > 1e-2 / (m * 1e-8)
    # zero target row: gradient exactly 0
    assert torch.equal(gt[3], torch.zeros_like(gt[3]))
    cf = cos_ref.cos_grad(fin, tin)
    assert torch.allclose(cf, gt, rtol=1e-10, atol=0)
    assert torch.equal(cf[3], gt[3])


# ------------------------------------------------------------------ the head's bounds against an emulation of its arithmetic
def _f32(v):
    return v.float().double()


def _chain(a, b):
    """a @ b as one fp32 FMA chain per element, k ascending (products exact in fp64, one rounding to fp32 per step)"""
    acc = torch.zeros(a.shape[0], b.shape[1], dtype=torch.float64)
    for k in range(a.shape[1]):
        acc = _f32(acc + a[:, k:k + 1] * b[k:k + 1, :])
    return acc


def _emulate(x, w, t, rows, g):
    """the documented arithmetic of osb_cos_head_fwd / osb_cos_head_bwd (csrc/cos_head.cu) on the CPU: f = x W in fp32 with k
    ascending, the row sums and the loss in fp64, (a, b) rounded to fp32, P = t W^T, G = W W^T and Q = x G as fp32 chains,
    dx = fmaf(a, P, fp32(b Q)) stored as split rows, dW from fp32 partials over row splits of the kernel's size merged in
    fp64, then dW = dsum_T + H W in fp64"""
    r = rows.long()
    m = r.shape[0]
    X, W, T = x.double()[r], w.double(), t.double()
    F = _chain(X, W)
    n1, ft, n2 = (F * F).sum(1).sqrt(), (F * T).sum(1), (T * T).sum(1).sqrt()
    loss = _f32((1 - ft / (n1.clamp_min(cos_ref.EPS) * n2.clamp_min(cos_ref.EPS))).sum() / m)
    a, b = cos_ref.cos_ab(n1, ft, n2, m, g)
    a, b = _f32(a), _f32(b)
    P, G = _chain(T, W.t()), _chain(W, W.t())
    Q = _chain(X, G)
    dx = _f32(a[:, None] * P + _f32(b[:, None] * Q))
    dx = R.split_decode(R.split_of(dx), dx.shape[1])
    s = cos_ref.dw_split_rows(m)
    V = torch.cat([_f32(a[:, None] * T), _f32(b[:, None] * X)], 1)
    dsum = torch.zeros(X.shape[1], V.shape[1], dtype=torch.float64)
    for r0 in range(0, m, s):
        acc = torch.zeros_like(dsum)
        for i in range(r0, min(m, r0 + s)):
            acc = _f32(acc + X[i][:, None] * V[i][None, :])
        dsum = dsum + acc
    c = W.shape[1]
    dW = _f32(dsum[:, :c] + dsum[:, c:] @ W)
    return dict(state=torch.stack([n1, ft, n2], 1), loss=loss, dx=dx, dW=dW)


def _within(got, ref):
    rs = cos_ref.ratios(got, ref)
    assert all(v <= 1 for v in rs.values()), rs
    return rs


def test_head_bounds_hold_for_the_emulated_arithmetic():
    for m, cin, c, edges in ((1100, 96, 768, False), (70, 384, 512, False), (300, 96, 768, True)):
        x, w, rows, t = cos_ref.case(m, cin, c, seed=m + cin, edges=edges)
        assert cos_ref.dw_splits(m) == (3 if m == 1100 else 1)
        got = _emulate(x, w, t, rows, 0.75)
        _within(got, cos_ref.head(x.double(), w, t.double(), rows, 0.75))
        if edges:
            assert float(got['state'][1, 0]) == 0.0 and 0 < float(got['state'][2, 0]) < cos_ref.EPS
            assert torch.equal(got['dx'][3], torch.zeros_like(got['dx'][3]))
            x[rows[4].long(), 7] = float('nan')
            assert torch.isnan(_emulate(x, w, t, rows, 0.75)['loss'])


def test_head_bounds_reject_mutated_references():
    """rows rolled by one, g = 1 for 0.75 and W after one Adam step (lr 1e-3: every weight moved by 1e-3) each put the
    emulated head outside the bounds of the outputs they change"""
    x, w, rows, t = cos_ref.case(300, 96, 768, seed=5)
    x64, t64 = x.double(), t.double()
    ref = cos_ref.head(x64, w, t64, rows, 0.75)
    got = _emulate(x, w, t, rows, 0.75)
    _within(got, ref)
    rolled = cos_ref.ratios(got, cos_ref.head(x64, w, t64, rows.roll(1), 0.75))
    assert all(rolled[k] > 1 for k in ('state', 'dx', 'dW')), rolled
    g1 = cos_ref.ratios(got, cos_ref.head(x64, w, t64, rows, 1.0))
    assert g1['state'] <= 1 and g1['loss'] <= 1 and g1['dx'] > 1 and g1['dW'] > 1, g1
    stepped = w.double() - 1e-3 * ref['dW'][0].sign()
    adam = cos_ref.ratios(got, cos_ref.head(x64, stepped, t64, rows, 0.75))
    assert all(adam[k] > 1 for k in ('state', 'dx', 'dW')), adam
