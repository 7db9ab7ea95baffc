"""The L1 distillation head kernels (osb_l1_head_fwd / osb_l1_head_bwd) through the C ABI against fp64, computed on exactly
the values the kernels multiply: the split rows decoded (x), the fp32 weights (W) and the fp16 targets widened (t).  The
reference and its per-element bounds are ``l1_ref.head`` (the derivation is in tests/l1_ref.py).  Every stored sign must equal
the fp64 sign of f - t wherever |f - t| exceeds the forward bound; the backward is held to fp64 on the stored signs.  Dyadic
operands make f exact, and with them the signs, the loss and both gradients are checked bit for bit, with planted ties,
NaN / +-inf targets and +-0.  The scale rule s = fp32(g fp32(1 / fp32(M C))) is checked against torch's own CUDA backward."""
import math

import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from tests import l1_ref as L
from tests import replay_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _case(m, cin, c, seed, exact=False):
    x, w, rows, t = (L.exact_case if exact else L.case)(m, cin, c, seed)
    return _split(x.to(DEV)), w.to(DEV), rows.to(DEV), t.to(DEV)


def _fwd(xs, cin, w, c, rows, t):
    n, m = xs.shape[0], rows.shape[0]
    ws_b = C.lib().osb_l1_head_workspace_bytes(m, cin, c)
    ws = torch.empty(ws_b, dtype=torch.uint8, device=DEV)
    signs = torch.full((m, c // 16), -1, dtype=torch.int32, device=DEV)       # code 3 everywhere: every word must be written
    loss = torch.full((1,), float('nan'), device=DEV)
    C.call('osb_l1_head_fwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(rows), m, C.ptr(t), C.ptr(signs), C.ptr(loss), C.ptr(ws),
           ws_b, C.stream_ptr())
    return signs, loss, ws, ws_b


def _run(xs, cin, w, c, rows, t, g=1.0):
    n, m = xs.shape[0], rows.shape[0]
    signs, loss, ws, ws_b = _fwd(xs, cin, w, c, rows, t)
    gt = torch.full((1,), g, device=DEV)
    dx = torch.full((n, 4 * cin), 0x7f, dtype=torch.uint8, device=DEV)    # poisoned: every row must be written
    dw = torch.full((cin, c), float('nan'), device=DEV)
    C.call('osb_l1_head_bwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(rows), m, C.ptr(signs), C.ptr(gt), C.ptr(dx), C.ptr(dw),
           C.ptr(ws), ws_b, C.stream_ptr())
    torch.cuda.synchronize()
    return signs, loss, dx, dw


def _check(xs, cin, w, c, rows, t, g=1.0):
    signs, loss, dx, dw = _run(xs, cin, w, c, rows, t, g)
    r = rows.long()
    S = L.decode(signs, c)
    x = R.split_decode(xs, cin)
    ref = L.head(x, w, t.double(), rows, signs=S, g=g)
    cert = L.certain(ref)
    assert bool((S[cert] == L.sgn(ref['d'][0])[cert]).all()), "a sign the forward bound decides is wrong"
    dxd = R.split_decode(dx, cin)
    got = dict(loss=loss[0], dx=dxd[r], dW=dw)
    for k, v in L.ratios(got, ref).items():
        assert v <= 1, (k, v)
    others = torch.ones(xs.shape[0], dtype=torch.bool, device=DEV)
    others[r] = False
    assert torch.equal(dx[others], torch.zeros_like(dx[others]))
    return signs, loss, dx, dw


@pytest.mark.parametrize('m,cin,c', [(1, 96, 768), (1, 32, 512), (63, 384, 512), (64, 96, 768), (65, 32, 768),
                                     (129, 96, 512), (511, 96, 768), (513, 384, 768), (32767, 96, 512), (20000, 96, 768),
                                     (20000, 384, 768), (160000, 96, 768)])
def test_against_fp64(m, cin, c):
    xs, w, rows, t = _case(m, cin, c, seed=m + cin + c)
    _check(xs, cin, w, c, rows, t, g=0.75)


def test_two_runs_are_bit_identical():
    xs, w, rows, t = _case(20000, 96, 768, seed=4)
    a = _run(xs, 96, w, 768, rows, t, 0.75)
    b = _run(xs, 96, w, 768, rows, t, 0.75)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.uint8), v.view(torch.uint8))


def _exact_expect(x, w, t, rows, g):
    """signs, loss (rows without a NaN target), dx rows and dW exactly as the documented arithmetic gives them on operands whose
    products are exact"""
    r = rows.long().cpu()
    m, c = r.shape[0], w.shape[1]
    D = x.double().cpu()[r] @ w.double().cpu() - t.double().cpu()
    S = L.sgn(D)
    s = L.scale(g, m, c)
    p = (S.double() @ w.double().cpu().t()).float()                    # sums of +-W in multiples of 1/8: exact
    v = torch.tensor(s, dtype=torch.float32) * p
    hi = v.bfloat16().float()
    dx = hi + (v - hi).bfloat16().float()
    dW = (s * (x.double().cpu()[r].t() @ S.double())).float()
    return D, S, dx, dW


@pytest.mark.parametrize('m,cin,c', [(40, 64, 768), (700, 96, 512), (3, 32, 512)])
def test_exact_probes(m, cin, c):
    x, w, rows, t = L.exact_case(m, cin, c, seed=m)
    xs = _split(x.to(DEV))
    assert torch.equal(R.split_decode(xs, cin).cpu(), x.double())   # x in multiples of 1/4: the split is exact
    signs, loss, dx, dw = _run(xs, cin, w.to(DEV), c, rows.to(DEV), t.to(DEV), g=0.75)
    D, S, dx_e, dW_e = _exact_expect(x, w, t, rows, 0.75)
    got_s = L.decode(signs, c)
    assert torch.equal(got_s, S)
    assert bool((got_s[0] == 0).all())                                   # ties: code 0
    if m > 2:
        assert bool((got_s[2, ::2] == 0).all())                          # d = 0 - (-0)
        assert int(got_s[1, 0]) == 0 and int(got_s[1, 1]) == -1 and int(got_s[1, 2]) == 1     # NaN, +inf, -inf targets
        assert math.isnan(float(loss))
    dxd = R.split_decode(dx, cin).cpu()
    assert torch.equal(dxd[rows.long().cpu()].float(), dx_e)
    assert torch.equal(dw.cpu(), dW_e)
    if m > 2:                                                            # without the NaN row the loss is exact
        keep = torch.ones(m, dtype=torch.bool)
        keep[1] = False
        loss2 = _fwd(xs, cin, w.to(DEV), c, rows[keep].to(DEV), t[keep].contiguous().to(DEV))[1]
        torch.cuda.synchronize()
        assert float(loss2) == float(np.float32(D[keep].abs().sum().item() / ((m - 1) * c)))


def test_infinite_target_makes_the_loss_inf():
    m, cin, c = 50, 32, 512
    x, w, rows, t = L.case(m, cin, c, seed=11)
    t[7, 9] = float('inf')
    signs, loss, dx, dw = _run(_split(x.to(DEV)), cin, w.to(DEV), c, rows.to(DEV), t.to(DEV), g=0.75)
    assert math.isinf(float(loss)) and float(loss) > 0
    assert int(L.decode(signs, c)[7, 9]) == -1
    assert bool(torch.isfinite(dw).all())


def test_nan_g_makes_every_gradient_nan():
    m, cin, c = 50, 32, 512
    xs, w, rows, t = _case(m, cin, c, seed=12)
    _, _, dx, dw = _run(xs, cin, w, c, rows, t, g=float('nan'))
    assert bool(torch.isnan(dw).all())
    assert bool(torch.isnan(R.split_decode(dx, cin)[rows.long()]).all())


@pytest.mark.parametrize('m,c,g', [(5, 768, 0.75), (7, 512, 0.75), (1, 768, 0.3), (3, 512, 0.3), (20000, 768, 0.75)])
def test_scale_rule_matches_torch_on_the_device(m, c, g):
    """torch's CUDA backward of L1Loss: every nonzero gradient is fp32(g * fp32(1 / fp32(M C))); at these (M, C, g) that
    differs from a true division in the last bit, so the rule is pinned, and the kernels use the same value"""
    f = torch.zeros(m, c, device=DEV, requires_grad=True)
    t = torch.ones(m, c, device=DEV, dtype=torch.float16)
    loss = torch.nn.L1Loss()(f, t.float())
    (g * loss).backward()
    got = f.grad.abs().unique()
    assert got.numel() == 1
    assert float(got) == L.scale(g, m, c)
    assert L.scale(g, m, c) != float(np.float32(np.float64(np.float32(g)) / (m * c)))
    # the kernels: f = 0 against t = 1 gives sgn = -1 everywhere; dW = s X^T (-1) exactly for one row of dyadic x
    x = torch.zeros(m + 1, 32)
    x[:, 0] = 1.0
    w = torch.zeros(32, c)
    rows = torch.arange(m, dtype=torch.int32)
    _, _, dx, dw = _run(_split(x.to(DEV)), 32, w.to(DEV), c, rows.to(DEV), t, g=g)
    s = L.scale(g, m, c)
    assert float(dw[0, 0]) == float(np.float32(-m * np.float64(s)))


def test_host_refusals():
    xs, w, rows, t = _case(100, 96, 768, seed=1)
    n, m, cin, c = xs.shape[0], rows.shape[0], 96, 768
    L_ = C.lib()
    ws_b = L_.osb_l1_head_workspace_bytes(m, cin, c)
    assert ws_b > 0
    for bad in [(0, cin, c), (m, 96 + 16, c), (m, 416, c), (m, cin, 640)]:
        assert L_.osb_l1_head_workspace_bytes(*bad) == 0
    ws = torch.empty(ws_b + 256, dtype=torch.uint8, device=DEV)
    signs = torch.empty((m, c // 16), dtype=torch.int32, device=DEV)
    loss = torch.empty(1, device=DEV)
    g = torch.ones(1, device=DEV)
    dx = torch.empty_like(xs)
    dw = torch.empty_like(w)

    def fwd(**kw):
        a = dict(x=C.ptr(xs), n=n, cin=cin, w=C.ptr(w), c=c, rows=C.ptr(rows), m=m, t=C.ptr(t), s=C.ptr(signs),
                 loss=C.ptr(loss), ws=C.ptr(ws), wsb=ws_b)
        a.update(kw)
        rc = L_.osb_l1_head_fwd(*a.values(), C.stream_ptr())
        return rc, (L_.osb_last_error() or b'').decode()

    def bwd(**kw):
        a = dict(x=C.ptr(xs), n=n, cin=cin, w=C.ptr(w), c=c, rows=C.ptr(rows), m=m, s=C.ptr(signs), g=C.ptr(g),
                 dx=C.ptr(dx), dw=C.ptr(dw), ws=C.ptr(ws), wsb=ws_b)
        a.update(kw)
        rc = L_.osb_l1_head_bwd(*a.values(), C.stream_ptr())
        return rc, (L_.osb_last_error() or b'').decode()

    assert fwd()[0] == 0 and bwd()[0] == 0
    torch.cuda.synchronize()
    for kw, msg in [(dict(m=n + 1), 'supervised rows'), (dict(cin=80), 'input channels'), (dict(c=640), 'output channels'),
                    (dict(t=None), 'target'), (dict(s=None), 'signs'), (dict(loss=None), 'loss'), (dict(wsb=ws_b - 1), 'workspace'),
                    (dict(ws=C.ptr(ws).value + 16), 'workspace'), (dict(s=C.ptr(signs).value + 4), 'aligned')]:
        rc, err = fwd(**kw)
        assert rc != 0 and msg in err, (kw, err)
    for kw, msg in [(dict(g=None), 'null g'), (dict(dx=C.ptr(xs)), 'overlap'), (dict(dw=C.ptr(ws)), 'overlap'),
                    (dict(s=None), 'signs'), (dict(wsb=0), 'workspace'), (dict(dx=C.ptr(dx).value + 8), 'aligned')]:
        rc, err = bwd(**kw)
        assert rc != 0 and msg in err, (kw, err)
