"""The cosine distillation head kernels (osb_cos_head_fwd / osb_cos_head_bwd) through the C ABI against fp64 torch, computed on
exactly the values the kernels multiply: the split rows decoded (x, ``replay_ref.split_decode``), the fp32 weights (W) and the
fp16 targets widened (t).  The reference and its per-element bounds are ``cos_ref.head`` (the derivation is in
tests/cos_ref.py).  Edge rows (``cos_ref.case``): a zero output row (x = 0), 0 < |f| < eps (x one small channel, so x W does
not cancel), a zero target row (dx exactly 0) and, in a call of its own, a NaN row (the loss is NaN)."""
import math

import pytest
import torch

from openscene_b200 import _cabi as C
from tests import cos_ref
from tests import replay_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _case(m, cin, c, seed, edges=False):
    x, w, rows, t = cos_ref.case(m, cin, c, seed, edges)
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
    r = rows.long()
    ref = cos_ref.head(R.split_decode(xs, cin), w, t.double(), rows, g)
    dxd = R.split_decode(dx, cin)
    got = dict(state=state, loss=loss[0], dx=dxd[r], dW=dw)
    for k, v in cos_ref.ratios(got, ref).items():
        assert v <= 1, (k, v)
    others = torch.ones(xs.shape[0], dtype=torch.bool, device=DEV)
    others[r] = False
    assert torch.equal(dx.view(xs.shape[0], -1)[others], torch.zeros_like(dx[others]))
    return state, loss, dx, dw, ref['dx'][0], r


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
    dxd = R.split_decode(dx, cin)
    assert dxd[r[2]].abs().max() > 1e-2 / (m * cos_ref.EPS)              # gradients of order 1 / (M eps)
    assert torch.equal(dxd[r[3]], torch.zeros_like(dxd[r[3]]))           # zero target row: gradient exactly 0
    # the NaN rule: one NaN in a supervised row makes the loss NaN
    x = R.split_decode(xs, cin).float()                                  # exact: hi + lo of an fp32 split
    x[r[4], 7] = float('nan')
    _, loss, _, _ = _run(_split(x), cin, w, c, rows, t)
    assert math.isnan(float(loss))
