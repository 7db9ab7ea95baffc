"""fp64 reference, per-score error bounds and dyadic probe operands for the open-vocabulary matching kernels
(csrc/match.cu, csrc/match_tc.cu), shared by tests/test_gpu_match_bounds.py, tests/test_gpu_match_exact.py, the two older
match tests and their CPU self-check tests/test_match_ref_cpu.py.  Every function runs on CPU or CUDA tensors.

The reference score is S[p, k] = sum_c a[p, c] t[k, c] in fp64, with `a` the fp16 operand run/evaluate.py:288-323 multiplies:
fp16(x) for distill / fusion, fp16(x / (|x| + 1e-5)) for the normalised products (norm, +1e-5 and division in fp16 for an
fp16 source, as torch does on an fp16 tensor).  A kernel score s satisfies, element by element (DESIGN.md section 2),

    |s - S| <= acc + E + 1/2 ulp16(|S| + acc + E)

* acc, the fp32 accumulation: tensor cores charge STEP = 18 x 2^-23 per K16 step over C/16 steps, CUDA cores 2^-24 per
  rounding on the longest path (C/32 FMAs of one lane + 5 shuffle adds), both of sum |a| |t| (+ E);
* E = sum_c e[p, c] |t[k, c]|, the operand error of the normalised products: the kernels compute x * rcp(d) (match_tc.cu) or
  x / d in fp32 with their own norm summation order, so their fp16 operand is a neighbour of the reference's: e = ulp16(a).
  For an fp16 source the fp16 norm itself may round to the neighbouring value (the fp32 sum lies within a few 2^-24 of an
  fp16 rounding boundary), which scales the row by up to 2^-10: e = 2 ulp16(a) + 2^-10 |a| there;
* the final rounding of the fp32 accumulator to fp16, half an ulp at the upper end of the interval.

The label rule of the non-vote kernels (k_match_tc, k_match_scores, k_match_ensemble, k_folded_head_finish): the lowest
column holding the largest non-NaN score; 0 when no score is above -inf (a row of NaN and -inf only).  smax is that largest
non-NaN score (-inf when there is none)."""
import math

import torch

STEP_TC = 18 * 2.0 ** -23           # one K16 step of wgmma into the fp32 accumulator (tests/replay_ref.py STEP)
U32 = 2.0 ** -24                    # one round-to-nearest fp32 operation
FP16_MAX_FINITE = 65504.0
FP16_OVERFLOW = 65520.0             # |x| >= this rounds to inf in fp16


def ulp16(v):
    """fp16 unit in the last place at |v| (2^-24 in the subnormal range and at 0)"""
    a = v.abs().double().clamp(min=2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def fp16_rn(v):
    """fp16 round-to-nearest of fp64 values that are exact in fp32 (one rounding)"""
    return v.float().half()


# ------------------------------------------------------------------------------------------------ operands
def operand(x, normalize):
    """the fp16 operand the reference multiplies, as fp64; x [n, C] fp32 or fp16"""
    if not normalize:
        return x.half().double()
    if x.dtype == torch.float16:
        nrm = x.double().norm(dim=1, keepdim=True).float().half()         # x.norm() on an fp16 tensor
        d = (nrm.float() + 1e-5).half()                                     # + 1e-5 on the fp16 norm
        return (x.float() / d.float()).half().double()                      # fp16 / fp16 -> fp16
    xd = x.double()
    return (xd / (xd.norm(dim=1, keepdim=True) + 1e-5)).float().half().double()


def operand_err(a, normalize, f16_source):
    """per-element bound e on |a_kernel - a| (0 when the operand is a plain fp16 rounding, which every route does alike)"""
    if not normalize:
        return torch.zeros_like(a)
    if f16_source:
        return 2 * ulp16(a) + 2.0 ** -10 * a.abs()
    return ulp16(a)


def acc_coeff(route, c):
    """accumulation charge per unit of sum |a| |t|: 'tc' (wgmma, C/16 K16 steps) or 'simt' (fp32 FMA chain + 5 adds)"""
    if route == 'tc':
        return (c // 16) * STEP_TC
    if route == 'simt':
        return (c // 32 + 5) * U32 * (1 + 2.0 ** -10)
    raise ValueError(route)


def reference(a, text, e=None):
    """(S, A, E) in fp64: S = a t^T, A = |a| |t|^T, E = e |t|^T"""
    t = text.double().to(a.device)
    at = t.abs()
    return a @ t.t(), a.abs() @ at.t(), (e @ at.t() if e is not None else torch.zeros(a.shape[0], t.shape[0],
                                                                                    dtype=torch.float64, device=a.device))


def bound(S, A, E, coeff):
    acc = coeff * (A + E)
    return acc + E + 0.5 * ulp16(S.abs() + acc + E)


def score_ratio(s, S, B):
    """max |s - S| / B over the elements (inf where the kernel returned a non-finite value for a finite S)"""
    err = (s.double() - S).abs()
    r = err / B.clamp(min=1e-300)
    r = torch.where(err == 0, torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def check_scores(s, x, inds, text, normalize, route, chunk=1 << 16):
    """every score of s [n_pts, K] (fp16) within its bound of the fp64 reference on the features x[inds]; returns the worst
    fraction of the bound used.  Chunked over rows so that large scenes fit."""
    f16 = x.dtype == torch.float16
    coeff = acc_coeff(route, x.shape[1])
    worst = 0.0
    n = s.shape[0]
    for r0 in range(0, n, chunk):
        rows = torch.arange(r0, min(n, r0 + chunk), device=x.device)
        xi = x[inds[rows]] if inds is not None else x[rows]
        a = operand(xi, normalize)
        S, A, E = reference(a, text, operand_err(a, normalize, f16))
        r = score_ratio(s[r0:r0 + len(rows)].to(x.device), S, bound(S, A, E, coeff))
        assert r <= 1.0, f"{route}: a score leaves its bound by {r:.3g}x (normalize={normalize}, fp16 source={f16})"
        worst = max(worst, r)
    return worst


# ------------------------------------------------------------------------------------------------ label rule
def label_rule(s):
    """(label, smax) of the non-vote kernels on their own scores s [n, K]: the lowest column holding the largest non-NaN
    score, 0 when no score is above -inf"""
    v = s.float()
    v = torch.where(torch.isnan(v), torch.full_like(v, -math.inf), v)
    m = v.max(dim=1).values
    hit = (v == m[:, None]) & (m[:, None] > -math.inf)
    k = torch.arange(v.shape[1], device=v.device).expand_as(v)
    lab = torch.where(hit, k, torch.full_like(k, v.shape[1])).min(dim=1).values
    lab = torch.where(lab == v.shape[1], torch.zeros_like(lab), lab)
    return lab, m


def check_labels(s, label, smax=None):
    lab, m = label_rule(s)
    label = label.to(s.device)
    assert bool(((label >= 0) & (label < s.shape[1])).all()), f"label outside [0, {s.shape[1]}): {label.min()} .. {label.max()}"
    bad = (label != lab).nonzero()
    assert bad.numel() == 0, f"label rule broken at row {int(bad[0])}: got {int(label[bad[0]])}, rule {int(lab[bad[0]])}"
    if smax is not None:
        assert torch.equal(smax.to(s.device).float(), m), "smax differs from the row maximum of the kernel's own scores"


# ------------------------------------------------------------------------------------------------ dyadic probes
def grid_unit(v, dim=1):
    """per row, the largest power of two of which every entry of v (fp64) is an integer multiple (inf for a zero row)"""
    m, e = torch.frexp(v.double())
    mi = (m.abs() * 2.0 ** 53).to(torch.int64)
    low = (mi & -mi).double()
    lsb = torch.where(mi != 0, torch.exp2(e.double() - 53) * low, torch.full_like(low, math.inf))
    return lsb.min(dim=dim).values


def exact_budget_bits(a, text):
    """log2 of the largest row budget max_k sum_c |a| |t| / u with u = grid_unit(a row) grid_unit(t): every product and every
    partial sum is a multiple of u, so below 2^24 u any fp32 accumulation order, and the tensor cores' alignment to the
    largest exponent, is exact"""
    t = text.double().to(a.device)
    u = grid_unit(a) * float(grid_unit(t.reshape(1, -1))[0])
    tot = (a.abs() @ t.abs().t()).max(dim=1).values
    ok = torch.isfinite(u) & (tot > 0)
    if not bool(ok.any()):
        return 0.0
    return float(torch.log2(tot[ok] / u[ok]).max())


def dyadic_text(k, c, gen, shared=16, support=64, device='cpu'):
    """text rows with entries +-2^-3 on `support` columns, the first `shared` of them common to every row and positive:
    every row has norm 1, so a point equal to a multiple of row j scores highest exactly at the rows equal to row j, and a
    point that is very negative on the shared columns drives every score of its row towards -inf"""
    t = torch.zeros(k, c, dtype=torch.float64)
    t[:, :shared] = 1.0
    for j in range(k):
        cols = shared + torch.randperm(c - shared, generator=gen)[:support - shared]
        t[j, cols] = torch.where(torch.rand(support - shared, generator=gen) < 0.5, -1.0, 1.0).double()
    return (t * 2.0 ** -3).half().to(device)


def dyadic_points(n, c, gen, norm_pow2=False):
    """fp64 point rows on a dyadic grid, exact in fp16.  Plain: entries {+-1, +-3, +-5, +-7} 2^e on ~40 % of the columns,
    e per row in [-8, 3].  norm_pow2: n1 entries +-2^e and n2 entries +-2^(e+1) with n1 + 4 n2 = 256, so |x| = 2^(e+4)
    exactly; every fourth row has |x| = 2^-5, the smallest norm whose fp16 +1e-5 still rounds back to it."""
    x = torch.zeros(n, c, dtype=torch.float64)
    if not norm_pow2:
        mag = torch.tensor([1.0, 3.0, 5.0, 7.0], dtype=torch.float64)
        v = mag[torch.randint(4, (n, c), generator=gen)]
        v = torch.where(torch.rand(n, c, generator=gen) < 0.5, -v, v) * (torch.rand(n, c, generator=gen) < 0.4)
        e = torch.randint(-8, 4, (n, 1), generator=gen).double()
        return v * torch.exp2(e)
    for i in range(n):
        n2 = int(torch.randint(0, 64, (1,), generator=gen))
        n1 = 256 - 4 * n2
        cols = torch.randperm(c, generator=gen)[:n1 + n2]
        vals = torch.cat([torch.ones(n1), torch.full((n2,), 2.0)]).double()
        sign = torch.where(torch.rand(n1 + n2, generator=gen) < 0.5, -1.0, 1.0).double()
        e = -9 if i % 4 == 0 else int(torch.randint(-9, 3, (1,), generator=gen))
        x[i, cols] = vals * sign * 2.0 ** e
    return x


def check_ensemble(s, label, fe, mask, f3, f2, inds, text, route, chunk=1 << 16):
    """the ensemble branch (matching.match_ensemble) against fp64: a point's 3-D / 2-D choice may differ from the fp64
    decision max S3 < max S2 only where the bound intervals of the two normalised maxima overlap; the ensemble feature is bit
    for bit the source row the kernel's own choice picked; the final scores are within the bound of that feature, and the
    labels follow the label rule.  Returns (worst fraction of the final scores' bound, disagreeing points, largest fp64 gap
    |max S3 - max S2| among them)."""
    coeff = acc_coeff(route, f3.shape[1])
    worst, n_dis, gap = 0.0, 0, 0.0
    n = s.shape[0]
    for r0 in range(0, n, chunk):
        rows = torch.arange(r0, min(n, r0 + chunk), device=f3.device)
        v = inds[rows] if inds is not None else rows
        x3, x2, m = f3[v], f2[v], mask[rows].to(f3.device)
        iv = []
        for xs, f16 in ((x3, False), (x2, True)):
            a = operand(xs, True)
            S, A, E = reference(a, text, operand_err(a, True, f16))
            B = bound(S, A, E, coeff)
            iv.append(((S - B).max(dim=1).values, S.max(dim=1).values, (S + B).max(dim=1).values))
        (lo3, s3, hi3), (lo2, s2, hi2) = iv
        dis = m != (s3 < s2)
        overlap = (lo3 <= hi2) & (lo2 <= hi3)
        assert not bool((dis & ~overlap).any()), f"{route}: a 3-D / 2-D choice contradicts separated bound intervals"
        if bool(dis.any()):
            n_dis += int(dis.sum())
            gap = max(gap, float((s3 - s2)[dis].abs().max()))
        chosen = torch.where(m[:, None], x2, x3.half())
        assert torch.equal(fe[rows].view(torch.int16), chosen.view(torch.int16)), f"{route}: ensemble feature is not the chosen row"
        worst = max(worst, check_scores(s[rows], fe[rows], None, text, False, route))
        check_labels(s[rows], label[rows])
    return worst, n_dis, gap
