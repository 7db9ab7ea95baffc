"""tests/match_ref.py without a GPU: the fp64 reference against the oracle's fp16 product (oracle/matching.py), the per-score
bound against fp32 sums taken in the orders the kernels use (the CUDA-core lane chains with their shuffle reduction, the
tensor cores' truncating alignment per K16 step) and in others, the dyadic probe operands under their exactness budget, and
negative controls that each break the bound: a score read from the neighbouring text row, a dropped K16 depth step, and an
operand left unrounded."""
import math

import pytest
import torch

from oracle import matching as om
from openscene_b200 import synth
from tests import match_ref as M


def _feats(n, c, seed, f16=False):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(n, c, generator=g) * (0.2 + torch.rand(n, 1, generator=g))
    return f.half() if f16 else f


def _text(k, c):
    return torch.from_numpy(synth.text_embeddings(k, c))


# ------------------------------------------------------------------------------------------------ fp32 summation models
def _products(a, t):
    """exact products a[p, c] t[k, c] (fp16 x fp16 is exact in fp32 and fp64): [n, K, C]"""
    return a[:, None, :] * t.double()[None, :, :]


def _f32(v):
    return v.float().double()


def simt_sum(p):
    """k_match_scores / k_match_ensemble: lane l chains fmaf over columns 2 (l + 32 j) + {0, 1}, j ascending, then a
    butterfly of __shfl_xor adds (every lane ends with the same value)"""
    n, k, c = p.shape
    q = p.view(n, k, c // 64, 32, 2)
    acc = torch.zeros(n, k, 32, dtype=torch.float64)
    for j in range(c // 64):
        for e in range(2):
            acc = _f32(acc + q[:, :, j, :, e])
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = _f32(acc + acc[:, :, lane ^ o])
    return acc[:, :, 0]


def _trunc_to(v, bits):
    """truncate toward zero to `bits` significant bits below the leading one"""
    e = torch.floor(torch.log2(v.abs().clamp(min=1e-300)))
    unit = torch.exp2(e - bits)
    return torch.where(v == 0, v, torch.trunc(v / unit) * unit)


def tc_sum(p):
    """one model of a wgmma K16 step: the 16 products and the accumulator aligned to the largest exponent and truncated to
    2^-23 of it, summed, and the sum truncated to fp32 (Fasi, Higham, Mikaitis, Pranesh 2021)"""
    n, k, c = p.shape
    acc = torch.zeros(n, k, dtype=torch.float64)
    for s in range(c // 16):
        terms = torch.cat([acc[..., None], p[..., 16 * s:16 * s + 16]], dim=-1)
        mx = terms.abs().max(dim=-1, keepdim=True).values
        unit = torch.exp2(torch.floor(torch.log2(mx.clamp(min=1e-300))) - 23)
        acc = _trunc_to((torch.trunc(terms / unit) * unit).sum(dim=-1), 23)
    return acc


def seq_sum(p, order):
    acc = torch.zeros(p.shape[:2], dtype=torch.float64)
    q = torch.gather(p, 2, order)
    for i in range(p.shape[2]):
        acc = _f32(acc + q[..., i])
    return acc


def pairwise_sum(p):
    width = 1 << (p.shape[-1] - 1).bit_length()
    q = torch.nn.functional.pad(p, (0, width - p.shape[-1]))
    while q.shape[-1] > 1:
        q = _f32(q[..., 0::2] + q[..., 1::2])
    return q[..., 0]


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('f16', [False, True])
@pytest.mark.parametrize('normalize', [False, True])
def test_reference_is_the_oracle_product(c, f16, normalize):
    """the operand is the oracle's (bit for bit when plain, within e when normalised), and the oracle's fp32 product lies
    within the bound of the fp64 reference"""
    x, t = _feats(300, c, 1, f16), _text(37, c)
    a = M.operand(x, normalize)
    a_or = (om._l2n(x) if normalize else x).half().double()
    e = M.operand_err(a, normalize, f16)
    if normalize:
        assert bool(((a - a_or).abs() <= e).all())
    else:
        assert torch.equal(a, a_or)
    S, A, E = M.reference(a_or, t)
    s = om._hmm(a_or.float(), t)
    assert M.score_ratio(s, S, M.bound(S, A, E, c * M.U32)) <= 1.0
    # one fp16 rounding of the fp64 sum almost everywhere: the reference is the oracle's arithmetic, not a neighbour of it
    assert (s == M.fp16_rn(S)).float().mean() > 0.99


@pytest.mark.parametrize('c', [512, 768])
def test_bound_covers_fp32_sums_in_every_order(c):
    x, t = _feats(48, c, 2), _text(23, c)
    a = M.operand(x, False)
    p = _products(a, t)
    S, A, E = M.reference(a, t)
    g = torch.Generator().manual_seed(3)
    mag = p.abs().argsort(dim=2)
    orders = {'ascending |p|': mag, 'descending |p|': mag.flip(2),
              'random': torch.stack([torch.randperm(c, generator=g) for _ in range(p.shape[0] * p.shape[1])]).view_as(p)}
    ratios = {'simt': M.score_ratio(M.fp16_rn(simt_sum(p)), S, M.bound(S, A, E, M.acc_coeff('simt', c))),
              'tc model': M.score_ratio(M.fp16_rn(tc_sum(p)), S, M.bound(S, A, E, M.acc_coeff('tc', c))),
              'pairwise': M.score_ratio(M.fp16_rn(pairwise_sum(p)), S, M.bound(S, A, E, M.acc_coeff('tc', c)))}
    for name, o in orders.items():
        ratios[name] = M.score_ratio(M.fp16_rn(seq_sum(p, o)), S, M.bound(S, A, E, M.acc_coeff('tc', c)))
    assert max(ratios.values()) <= 1.0, ratios
    # the accumulation models really are different sums (the bound is not tested on one order only)
    assert not torch.equal(tc_sum(p), simt_sum(p))


def test_the_tc_model_loses_what_the_bound_charges():
    """the truncating model's own error, before the fp16 rounding, stays within the accumulation charge and uses a visible
    part of it on adversarial magnitudes (one dominant product per K16 slice)"""
    c = 768
    g = torch.Generator().manual_seed(4)
    x = torch.randn(16, c, generator=g) * 1e-2
    x[:, ::16] = 30.0
    t = _text(11, c)
    a = M.operand(x, False)
    p = _products(a, t)
    S, A, _ = M.reference(a, t)
    err = (tc_sum(p) - S).abs()
    charge = M.acc_coeff('tc', c) * A
    assert bool((err <= charge).all())
    assert float((err / charge).max()) > 1e-3


@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('norm_pow2', [False, True])
def test_dyadic_probes_are_exact_in_any_order(c, norm_pow2):
    g = torch.Generator().manual_seed(5)
    t = M.dyadic_text(97, c, g)
    assert torch.allclose(t.double().norm(dim=1), torch.ones(97, dtype=torch.float64))
    x = M.dyadic_points(40, c, g, norm_pow2)
    assert torch.equal(x.half().double(), x)                                  # exact in fp16
    if norm_pow2:
        nrm = x.norm(dim=1)
        assert torch.equal(torch.exp2(torch.round(torch.log2(nrm))), nrm) and float(nrm.min()) == 2.0 ** -5
        a = M.operand(x.half(), True)
        assert torch.equal(a, x / nrm[:, None])                               # d = |x| exactly: x rcp(d) = x / d
    else:
        a = x
    # planted: a multiple of a text row, a row of fp16 maxima on the shared columns (every score overflows to -inf)
    big = torch.zeros(2, c, dtype=torch.float64)
    big[0] = t[3].double() * 2.0 ** 16
    big[1, :16] = -M.FP16_MAX_FINITE
    a = torch.cat([a, big])
    bits = M.exact_budget_bits(a, t)
    assert bits < 24, bits
    p = _products(a, t)
    S = a @ t.double().t()
    for s in (simt_sum(p), tc_sum(p), pairwise_sum(p), seq_sum(p, p.abs().argsort(dim=2).flip(2))):
        assert torch.equal(s, S)
    ref = M.fp16_rn(S)
    assert bool(torch.isinf(ref[-1]).all() and (ref[-1] < 0).all())           # all -inf
    assert math.isinf(float(ref[-2, 3])) and float(ref[-2, 3]) > 0


def test_grid_unit_and_budget():
    v = torch.tensor([[0.75, -0.5, 0.0], [3.0, 6.0, 0.0], [0.0, 0.0, 0.0]], dtype=torch.float64)
    assert M.grid_unit(v).tolist() == [0.25, 1.0, math.inf]
    t = torch.tensor([[0.125, -0.25, 0.5]], dtype=torch.float16)
    # row 1: sum |a||t| = 3/8 + 6/4 = 1.875, unit 1 * 1/8 -> 15
    assert M.exact_budget_bits(v[1:2], t) == pytest.approx(math.log2(15))


def test_label_rule():
    nan, inf = math.nan, math.inf
    s = torch.tensor([[1.0, 3.0, nan, 3.0],
                      [nan, nan, nan, nan],
                      [-inf, -inf, -inf, -inf],
                      [nan, -inf, nan, -inf],
                      [-0.0, 0.0, -1.0, 0.0],
                      [inf, nan, inf, 2.0]]).half()
    lab, m = M.label_rule(s)
    assert lab.tolist() == [1, 0, 0, 0, 0, 0]
    assert m[0] == 3 and m[1] == -inf and m[2] == -inf and m[3] == -inf and m[4] == 0 and m[5] == inf
    M.check_labels(s, lab, m)
    with pytest.raises(AssertionError):
        M.check_labels(s, torch.tensor([3, 0, 0, 0, 0, 0]))                   # the last maximum
    with pytest.raises(AssertionError):
        M.check_labels(s, torch.tensor([1, 0x7fffffff, 0, 0, 0, 0]))          # outside [0, K)


# ------------------------------------------------------------------------------------------------ negative controls
@pytest.mark.parametrize('route', ['tc', 'simt'])
@pytest.mark.parametrize('normalize', [False, True])
def test_shifted_text_row_and_dropped_depth_step_break_the_bound(route, normalize):
    c = 768
    x, t = _feats(64, c, 6), _text(40, c)
    a = M.operand(x, normalize)
    S, A, E = M.reference(a, t, M.operand_err(a, normalize, False))
    B = M.bound(S, A, E, M.acc_coeff(route, c))
    assert M.score_ratio(M.fp16_rn(S), S, B) <= 1.0
    shifted = S.clone()
    shifted[:, 7] = S[:, 8]                                                   # one pass loaded at row offset +1
    assert M.score_ratio(M.fp16_rn(shifted), S, B) > 1
    keep = torch.ones(c, dtype=torch.float64)
    keep[48:64] = 0                                                           # the h = 3 K16 step of the first chunk
    dropped = (a * keep) @ t.double().t()
    assert M.score_ratio(M.fp16_rn(dropped), S, B) > 1


@pytest.mark.parametrize('route', ['tc', 'simt'])
def test_unrounded_operand_breaks_the_bound(route):
    """pairs of equal fp16 values against text entries of opposite sign: the rounded operand scores exactly 0, the operand
    left in fp32 (each entry 0.4 ulp16 off, signed like its text entry) scores 0.4 sum ulp16(a)|t|, above the charge"""
    c = 768
    g = torch.Generator().manual_seed(7)
    v = (1 + torch.randint(1, 1024, (8, c // 2), generator=g).double() / 1024).repeat_interleave(2, dim=1)
    t = (torch.rand(5, c // 2, generator=g).double() * 0.1 + 0.01).repeat_interleave(2, dim=1)
    t[:, 1::2] *= -1
    t = t.half()
    x = (v + 0.4 * M.ulp16(v) * torch.sign(t[0].double())).float()
    a = M.operand(x, False)
    assert torch.equal(a, v)
    S, A, E = M.reference(a, t)
    assert float(S[:, 0].abs().max()) == 0.0
    B = M.bound(S, A, E, M.acc_coeff(route, c))
    unrounded = x.double() @ t.double().t()
    assert M.score_ratio(M.fp16_rn(unrounded[:, :1]), S[:, :1], B[:, :1]) > 1
