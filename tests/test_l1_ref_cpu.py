"""The L1 head's fp64 restatement (tests/l1_ref.py) against torch's CPU autograd, and its bounds against an fp32 emulation of
the documented kernel arithmetic and against mutated restatements.  No GPU."""
import math

import pytest
import torch

from openscene_b200 import distill
from tests import l1_ref as L
from tests import replay_ref as R


def _edge_rows(c, seed=0):
    """(f fp32 [8, C], t fp16 [8, C]): random rows, with NaN, +inf and -inf targets, exact ties f == t, and d = +-0"""
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(8, c, generator=g)
    t = (f + 0.3 * torch.randn(8, c, generator=g)).half()
    f[1] = t[1].float()                                   # ties: d = 0 everywhere
    t[2, :5] = torch.tensor([float('nan'), float('inf'), float('-inf'), 0.0, -0.0]).half()
    f[2, 3], f[2, 4] = -0.0, 0.0                          # d = -0 - 0 and 0 - (-0)
    f[3, 7] = float('nan')
    return f, t


@pytest.mark.parametrize('c', [512, 768])
def test_sign_pattern_equals_torch_autograd(c):
    f, t = _edge_rows(c, seed=c)
    fr = f.clone().requires_grad_(True)
    loss = distill.distill_loss(fr, t, 'l1')
    assert type(loss.grad_fn).__name__ == 'MeanBackward0'
    (0.75 * loss).backward()
    gd = fr.grad
    d = f - t.float()
    s = L.sgn(d)
    assert torch.equal(torch.sign(gd).to(torch.int8), s)
    assert bool((gd[s == 0] == 0).all())                 # NaN, ties and +-0: exactly zero gradient
    assert int((s == 0).sum()) >= c + 4
    mags = gd[s != 0].abs().unique()
    assert mags.numel() == 1 and math.isclose(float(mags), L.scale(0.75, 8, c), rel_tol=1e-6)
    # the loss: NaN with a NaN element, and the restatement's value on the rows without one
    assert math.isnan(float(loss.detach()))
    ok = torch.tensor([0, 1, 4, 5, 6, 7])
    ref = (f[ok].double() - t[ok].double()).abs().mean()
    got = distill.distill_loss(f[ok], t[ok], 'l1')
    assert math.isclose(float(got), float(ref), rel_tol=1e-6)
    # an infinite d makes the loss inf
    inf_rows = torch.tensor([0, 2])
    t2 = t.clone()
    t2[2, 0] = 0
    assert math.isinf(float(distill.distill_loss(f[inf_rows], t2[inf_rows], 'l1')))


def test_pack_and_decode_round_trip():
    g = torch.Generator().manual_seed(3)
    s = torch.randint(-1, 2, (5, 768), generator=g).to(torch.int8)
    w = L.pack(s)
    assert w.shape == (5, 48) and w.dtype == torch.int32
    assert torch.equal(L.decode(w, 768), s)
    # element j: bits 2 (j % 16) of word j / 16; code 1 = +1, 2 = -1
    one = torch.zeros(1, 512, dtype=torch.int8)
    one[0, 17], one[0, 31] = 1, -1
    assert int(L.pack(one)[0, 1]) & 0xFFFFFFFF == (1 << 2) | (2 << 30)
    with pytest.raises(AssertionError, match='code 3'):
        L.decode(torch.full((1, 32), -1, dtype=torch.int32), 512)


def _x_split(x):
    """x as the head reads it: through the split of its fp32 rows"""
    return R.split_decode(R.split_of(x), x.shape[1])


@pytest.mark.parametrize('m,cin,c', [(37, 64, 512), (600, 32, 768)])
def test_emulation_stays_inside_the_bounds(m, cin, c):
    x, w, rows, t = L.case(m, cin, c, seed=m + c)
    xd = _x_split(x)
    loss, S, dx, dW = L.emulate(xd, w, t, rows, g=0.75)
    ref = L.head(xd, w, t.double(), rows, signs=S, g=0.75)
    cert = L.certain(ref)
    assert bool((S[cert] == L.sgn(ref['d'][0])[cert]).all())
    assert cert.float().mean() > 0.95
    r = L.ratios(dict(loss=loss, dx=dx, dW=dW), ref)
    assert all(v <= 1 for v in r.values()), r
    # torch's own loss (fp32 sum) agrees closely
    assert math.isclose(float(L.l1_loss(xd[rows.long()].float() @ w, t)), float(ref['loss'][0]), rel_tol=1e-5)


def test_exact_operands_give_exact_signs_and_loss():
    m, cin, c = 40, 64, 768
    x, w, rows, t = L.exact_case(m, cin, c, seed=5)
    loss, S, dx, dW = L.emulate(x, w, t, rows, g=0.75)
    D = x.double()[rows.long()] @ w.double() - t.double()
    assert torch.equal(S, L.sgn(D))
    assert bool((S[0] == 0).all()) and bool((S[2, ::2] == 0).all()) and int(S[1, 0]) == 0
    assert int(S[1, 1]) == -1 and int(S[1, 2]) == 1
    assert math.isnan(float(loss))
    fin = torch.ones(m, dtype=torch.bool)
    fin[1] = False
    loss2, *_ = L.emulate(x, w, t[fin], rows[fin], g=0.75)
    assert float(loss2) == float(torch.tensor(float(D[fin].abs().sum() / ((m - 1) * c)), dtype=torch.float32))


def _mutants(x, w, t, rows, S, D):
    nan = torch.isnan(D)
    tie = (D == 0)
    m, c = S.shape
    yield 'sign(0) = +1', L.head(x, w, t, rows, signs=torch.where(tie, torch.ones_like(S), S), g=0.75)
    yield 'gradient at NaN', L.head(x, w, t, rows, signs=torch.where(nan, torch.ones_like(S), S), g=0.75)
    yield 'scale 1/M', L.head(x, w, t, rows, signs=S, g=0.75, s=0.75 / m)
    yield 'g = 1', L.head(x, w, t, rows, signs=S, g=1.0)
    yield 'rows rolled', L.head(x, w, t, rows.roll(1), g=0.75)


def test_mutated_restatements_fall_outside_the_bounds():
    m, cin, c = 40, 64, 512
    x, w, rows, t = L.exact_case(m, cin, c, seed=7)
    loss, S, dx, dW = L.emulate(x, w, t, rows, g=0.75)
    D = x.double()[rows.long()] @ w.double() - t.double()
    good = L.head(x, w, t.double(), rows, signs=S, g=0.75)
    assert all(v <= 1 for v in L.ratios(dict(dx=dx, dW=dW), good).values())
    for name, ref in _mutants(x, w, t.double(), rows, S, D):
        r = L.ratios(dict(dx=dx, dW=dW), ref)
        assert max(r.values()) > 1, (name, r)
