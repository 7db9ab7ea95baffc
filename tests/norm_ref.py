"""fp64 references, per-element error bounds, launch plans and exact probes for the train-mode BatchNorm kernels
(csrc/bn_train.cu) and the softmax cross-entropy head (csrc/ce_head.cu), shared by tests/test_gpu_bn_exact.py,
tests/test_gpu_bn_batch_stats.py, tests/test_gpu_bn_backward.py, tests/test_gpu_ce_head.py and their CPU self-check
tests/test_norm_ref_cpu.py.  Every function runs on CPU or CUDA tensors; split rows are decoded with
``replay_ref.split_decode`` (hi + lo, exact in fp64).

Launch plans (restated from the host code, so that bounds carry the real accumulation depth):
  statistics and backward reduce: ``bn_row_blocks(n) = min(ceil(n / 512), 1024)`` blocks of ``ceil(n / blocks)`` rows, 32 row
  slots per block each summing every 32nd row in fp64, a fixed-order merge of the 32 slots, then one block merging the block
  partials in 8 slots (``b = slot, slot + 8, ...``) and the 8 slot sums:  depth = ceil(rows / 32) + 32 + ceil(blocks / 8) + 8.
  CE head: ``ce_row_blocks(n) = min(ceil(n / 256), 1024)``, ``ce_splits(n) = min(ceil(n / 1024), 128)`` splits of
  ``ceil(n / splits)`` rows for dW, walked in tiles of ``CE_TILE = 64`` rows by one fp32 FMA chain per (channel, class).

Bounds, u = 2^-53 (fp64), and hu(v) = half an fp32 ulp at |v| (<= 2^-24 |v|, the error of one round-to-nearest to fp32):
* statistics: the shifted sums ``t1 = sum (x - x0)``, ``t2 = sum (x - x0)^2`` (x0 = row 0) are off by at most
  (depth + 3) u S1 and (depth + 3) u S2 (S1 = sum |x - x0|, S2 = sum (x - x0)^2); that error is carried through
  dm = t1 / n, var = t2 / n - dm^2, mean = x0 + dm, invstd = (var + eps)^-1/2, scale = w invstd, shift = b - mean scale and the
  running-buffer update to first order (``stats_bounds``), and each stored value adds one fp32 rounding hu(value).  In
  practice: one half-ulp of fp32, plus a few fp64 units where dm^2 cancels against t2 / n.
* apply, judged against the fp64 statistics (not the kernel's own fp32 scale / shift, so the hand-off is measured):
  hu(|z scale| + |shift|) for the fp32 scale / shift (two roundings, charged 2^-24 each), hu of the FMA and of the residual add
  (and of the residual's own FMA and scale / shift), then 2^-17 |y| for the split store.
* backward reduce: sums / dweight / dbias, per channel: (depth + 4) u sum |g'| |x^| (fp64) and one fp32 rounding; in
  accumulate mode the one rounding is of prev + t (a double rounding prev + fp32(t) is not within it).
* dz: 2^-21 |a| (|g'| + |sum g' / n| + |x^ sum g' x^ / n|) + 2^-17 |dz| on the operands the launch read (fp32 mean, invstd,
  sums); g': exact (mode 1), one fp32 rounding of prev + g' (mode 2), each then split-stored.
* CE dW: (rows per split + 5) 2^-24 sum_r |x_rk| |d_rc|  +  sum_r |x_rk| eps_r |p_rc s|, eps_r = 2^-18 (max_c sum_k |x_k w_kc|
  + |lse_r|) the relative error the fp32 logits and the fp32 lse carry into softmax (s = g / n_valid); the +5 covers the fp32
  rounding of d itself (exp, the one-hot subtraction, the scale) and the final rounding of the fp64 merge.

Exact probes: values on a short dyadic grid, n a power of two, every channel built as +-s pairs around a dyadic mean (or, with
the pivot row 0 deliberately far from the mean, as +-A outliers over rows at the mean), eps = 0 and var a power of four, so that
sqrt and 1 / sqrt are exact and every fp64 / fp32 step of the kernels is exact while the exactness budget
log2(max |term| / grid) stays below 24 (``replay_ref.exact_budget_bits``): every output must then equal its exact value."""
import math
from fractions import Fraction

import torch

from tests import replay_ref as R

U64 = 2.0 ** -53
U32 = 2.0 ** -24
OUT_SPLIT = 2.0 ** -17

# ------------------------------------------------------------------ launch plans (csrc/bn_train.cu, csrc/ce_head.cu)
BN_ROWS_PER_BLOCK, BN_MAX_ROW_BLOCKS, BN_ROW_SLOTS, BN_MERGE_SLOTS = 512, 1024, 32, 8
CE_THREADS, CE_MAX_ROW_BLOCKS, CE_SPLIT_ROWS, CE_MAX_SPLITS, CE_TILE = 256, 1024, 1024, 128, 64


def cdiv(a, b):
    return -(-a // b)


def bn_row_blocks(n):
    return min(cdiv(n, BN_ROWS_PER_BLOCK), BN_MAX_ROW_BLOCKS)


def bn_block_rows(n):
    """rows of one partial block (the last may be shorter or empty)"""
    return cdiv(n, bn_row_blocks(n))


def bn_depth(n):
    """longest chain of fp64 adds one row's term passes through: its slot's rows, the 32-slot merge, the finalize slot's
    blocks and the 8-slot merge"""
    return cdiv(bn_block_rows(n), BN_ROW_SLOTS) + BN_ROW_SLOTS + cdiv(bn_row_blocks(n), BN_MERGE_SLOTS) + BN_MERGE_SLOTS


def apply_grid(n, c):
    """(row blocks, channel blocks) of k_bn_apply / k_bn_bwd_apply (grid-stride over rows of 32 slots)"""
    return min(cdiv(n, BN_ROW_SLOTS), max(1, 132 * 8 // (c // 32))), c // 32


def ce_row_blocks(n):
    return min(cdiv(n, CE_THREADS), CE_MAX_ROW_BLOCKS)


def ce_splits(n):
    return min(cdiv(n, CE_SPLIT_ROWS), CE_MAX_SPLITS)


def ce_split_rows(n):
    return cdiv(n, ce_splits(n))


# ------------------------------------------------------------------ fp32 rounding helpers
def hu(v):
    """half an fp32 ulp at |v| (fp64 tensor), i.e. the largest error of one round-to-nearest of a value of that magnitude;
    2^-150 (half the smallest subnormal) at and below the subnormal range"""
    v = v.double().abs()
    _, e = torch.frexp(v)                         # v = m 2^e, m in [0.5, 1)
    h = torch.ldexp(torch.ones_like(v), (e - 25).clamp(min=-150))
    return torch.where(v > 0, h, torch.full_like(v, 2.0 ** -150))


def f32(v):
    return v.float().double()


# ------------------------------------------------------------------ references: statistics
def bn_stats(x, w, b, eps):
    """fp64 batch statistics of x [n, c] (fp64): dict of mean, var (biased), invstd, scale, shift and the magnitudes the
    bounds need (S1, S2 of the shifted sums, n)"""
    n = x.shape[0]
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    invstd = 1.0 / torch.sqrt(var + eps)
    scale = w.double() * invstd
    shift = b.double() - mean * scale
    d = x - x[0]
    return dict(mean=mean, var=var, invstd=invstd, scale=scale, shift=shift, n=n, eps=eps,
                S1=d.abs().sum(0), S2=(d * d).sum(0), x0=x[0], w=w.double(), b=b.double())


def bn_running(rm, rv, nbt, st, momentum):
    """torch.nn.modules.batchnorm's running-buffer update: (running_mean, running_var, num_batches_tracked, factor);
    momentum None: the cumulative factor 1 / num_batches_tracked, read after the increment; the variance is unbiased"""
    n = st['n']
    tracked = int(nbt) + 1
    m = 1.0 / tracked if momentum is None else momentum
    rm_new = (1.0 - m) * rm.double() + m * st['mean']
    rv_new = (1.0 - m) * rv.double() + m * st['var'] * n / (n - 1)
    return rm_new, rv_new, tracked, m


def stats_bounds(st, rm=None, rv=None, m=None):
    """per-channel bounds of every fp32 output of osb_bn_batch_stats(_save): dict name -> bound (fp64 [c])"""
    n, eps = st['n'], st['eps']
    depth = bn_depth(n)
    mean, var, istd, sc, sh = st['mean'], st['var'], st['invstd'], st['scale'], st['shift']
    dm = mean - st['x0']
    e_t1 = (depth + 3) * U64 * st['S1']
    e_t2 = (depth + 3) * U64 * st['S2']
    e_dm = e_t1 / n + U64 * dm.abs()
    e_var = e_t2 / n + 2 * U64 * st['S2'] / n + 2 * dm.abs() * e_dm + 3 * U64 * dm * dm + U64 * var
    e_mean = e_dm + U64 * mean.abs()
    e_istd = istd * (e_var / (2 * (var + eps)) + 4 * U64)
    e_sc = st['w'].abs() * e_istd + U64 * sc.abs()
    e_sh = mean.abs() * e_sc + sc.abs() * e_mean + 2 * U64 * (mean * sc).abs() + U64 * sh.abs()
    slack = 1 + 2.0 ** -20
    out = dict(mean=hu(mean) * slack + e_mean, invstd=hu(istd) * slack + e_istd, scale=hu(sc) * slack + e_sc,
               shift=hu(sh) * slack + e_sh, var=e_var, e_mean=e_mean, e_var=e_var, e_sc=e_sc, e_sh=e_sh)
    if rm is not None:
        e_rm = m * e_mean + 4 * U64 * ((1 - m) * rm.double().abs() + m * mean.abs())
        uv = var * n / (n - 1)
        e_rv = m * e_var * n / (n - 1) + 6 * U64 * ((1 - m) * rv.double().abs() + m * uv)
        rm_new = (1.0 - m) * rm.double() + m * mean
        rv_new = (1.0 - m) * rv.double() + m * uv
        out['running_mean'] = hu(rm_new) * slack + e_rm
        out['running_var'] = hu(rv_new) * slack + e_rv
    return out


# ------------------------------------------------------------------ references: apply
def bn_apply(z, st, res=None, res_st=None, relu=True):
    """y = act(z scale + shift + r) in fp64 on the fp64 statistics; r = none | res | res res_scale + res_shift.
    Returns (y, bound) with the bound of the module docstring."""
    sc, sh = st['scale'], st['shift']
    eb = stats_bounds(st)
    t = z * sc + sh
    # the fp32 scale / shift, the product (charged even though fmaf does not round it) and the FMA's rounding
    err = (z.abs() * eb['scale'] + eb['shift']) + hu(z * sc) * 1.0001 + hu(t) * 1.0001
    if res is None:
        r = torch.zeros_like(t)
    elif res_st is None:
        r = res
    else:
        rb = stats_bounds(res_st)
        r = res * res_st['scale'] + res_st['shift']
        err = err + res.abs() * rb['scale'] + rb['shift'] + hu(res * res_st['scale']) * 1.0001 + hu(r) * 1.0001
    pre = t + r
    if res is not None:
        err = err + hu(pre.abs() + err) * 1.0001
    y = torch.relu(pre) if relu else pre
    err = err * (1 + 2.0 ** -20) + OUT_SPLIT * (pre.abs() + err)
    return y, err


def relu_nan(v):
    """torch.relu: NaN passes through"""
    return torch.where(v < 0, torch.zeros_like(v), v)


# ------------------------------------------------------------------ references: backward
def bn_backward(y, g, z, mean, invstd, w, n=None):
    """the backward of act(BN(z) + r) on the operands one launch pair reads (fp64 of the fp32 saved mean / invstd / weight):
    g' = g where not y <= 0 (torch's threshold_backward; y None: no ReLU), x^ = (z - mean) invstd,
    t1 = sum g' (dbias), t2 = sum g' x^ (dweight), and the magnitudes of the bound"""
    n = z.shape[0] if n is None else n
    mean, invstd, w = mean.double(), invstd.double(), w.double()
    gp = g if y is None else torch.where(y <= 0, torch.zeros_like(g), g)
    xh = (z - mean) * invstd
    t1, t2 = gp.sum(0), (gp * xh).sum(0)
    A1, A2 = gp.abs().sum(0), (gp * xh).abs().sum(0)
    return dict(gp=gp, xh=xh, t1=t1, t2=t2, A1=A1, A2=A2, n=n, w=w, invstd=invstd)


def reduce_bounds(bw, prev_dw=None, prev_db=None):
    """bounds of sums [2c] / dweight / dbias; with prev (accumulate) the rounding is of prev + t"""
    d = bn_depth(bw['n']) + 4
    e1, e2 = d * U64 * bw['A1'], d * U64 * bw['A2'] * (1 + 4 * U64)
    db = bw['t1'] if prev_db is None else prev_db.double() + bw['t1']
    dw = bw['t2'] if prev_dw is None else prev_dw.double() + bw['t2']
    return dict(sums=torch.cat([hu(bw['t1'].abs() + e1) + e1, hu(bw['t2'].abs() + e2) + e2]),
                dbias=hu(db.abs() + e1) + e1, dweight=hu(dw.abs() + e2) + e2, db_ref=db, dw_ref=dw)


def bn_dz(bw, sums):
    """dz = a (g' - b - x^ k2) with a = weight invstd, b = sum g' / n, k2 = sum g' x^ / n from the sums the launch read
    (fp32 [2c]); returns (dz, bound)"""
    n, c = bw['n'], bw['gp'].shape[1]
    a = bw['w'] * bw['invstd']
    b, k2 = sums[:c].double() / n, sums[c:].double() / n
    gp, xh = bw['gp'], bw['xh']
    dz = a * (gp - b - xh * k2)
    tol = 2.0 ** -21 * a.abs() * (gp.abs() + b.abs() + (xh * k2).abs()) + OUT_SPLIT * dz.abs()
    return dz, tol


# ------------------------------------------------------------------ references: cross-entropy head
def ce_forward(x, w, row_map, labels, ignore):
    """x [n, cin] fp64 in internal row order, w [cin, C]; labels in caller order, internal row r has caller row row_map[r].
    Returns dict z, lse, pred (caller order: the first NaN, else the first maximum), nll, loss, n_valid, labelled, lab"""
    z = x @ w.double()
    lse = torch.logsumexp(z, 1)
    rm = row_map.long()
    lab = labels.long()[rm]
    labelled = lab != ignore
    nv = int(labelled.sum())
    pred_int = first_argmax(z)
    pred = torch.empty(labels.shape[0], dtype=torch.int64, device=z.device)
    pred[rm] = pred_int
    zl = z.gather(1, lab.clamp(0, z.shape[1] - 1)[:, None])[:, 0]
    nll = torch.where(labelled, lse - zl, torch.zeros_like(lse))
    loss = nll.sum() / nv if nv else torch.tensor(float('nan'), dtype=torch.float64, device=z.device)
    return dict(z=z, lse=lse, pred=pred, pred_int=pred_int, nll=nll, loss=loss, n_valid=nv, labelled=labelled, lab=lab)


def first_argmax(z):
    """torch's max(1)[1] rule: the first NaN of a row, else the first maximum (0 for a row of -inf)"""
    isn = torch.isnan(z)
    zz = torch.where(isn, torch.full_like(z, float('inf')), z)
    col = torch.arange(z.shape[1], device=z.device)
    best = zz.max(1, keepdim=True).values
    hit = (zz == best) & (isn | ~isn.any(1, keepdim=True))
    idx = torch.where(hit, col, torch.full_like(col, z.shape[1])).min(1).values
    return torch.where(idx == z.shape[1], torch.zeros_like(idx), idx)


def ce_backward(x, w, fw, g):
    """d = (softmax(z) - onehot) g / n_valid on labelled rows, dx = d w^T, dW = x^T d, with the bound terms of dW / dx"""
    z, lse, labelled, lab = fw['z'], fw['lse'], fw['labelled'], fw['lab']
    nv = fw['n_valid']
    c = z.shape[1]
    w64 = w.double()
    s = g / nv if nv else 0.0
    p = torch.softmax(z, 1) * s * labelled[:, None]
    d = p - torch.nn.functional.one_hot(lab.clamp(0, c - 1), c).double() * s * labelled[:, None]
    dx, dW = d @ w64.t(), x.t() @ d
    zabs = (x.abs() @ w64.abs()).max(1).values
    eps = 2.0 ** -18 * (zabs + lse.abs())
    return dict(d=d, p=p, dx=dx, dW=dW, eps=eps, s=s)


def ce_dw_bound(x, bw, n):
    depth = ce_split_rows(n) + 5
    return depth * U32 * (x.abs().t() @ bw['d'].abs()) + x.abs().t() @ (bw['eps'][:, None] * bw['p'].abs())


def ce_dx_bound(w, bw):
    w64 = w.double().abs()
    return (OUT_SPLIT * bw['dx'].abs() + 2.0 ** -22 * (bw['d'].abs() @ w64.t())
            + bw['eps'][:, None] * (bw['p'].abs() @ w64.t()))


# ------------------------------------------------------------------ exact probes
def probe_stats_rows(n, c, generator=None, far_pivot=None):
    """fp32 [n, c] probe rows (n a power of two) and the exact (mean, sigma) per channel: channel values are +-s pairs around
    a dyadic mean (var = s^2), or -- in the far-pivot channels -- rows at the mean except 2 (n = 2^odd) or 4 (n = 2^even)
    outliers +-A with row 0 = mean + A, var = k A^2 / n a power of four.  s, A powers of two, means on the 2^-4 grid."""
    k = int(math.log2(n))
    assert 2 ** k == n and n >= 2
    gen = generator
    mu = (torch.randint(-2 ** 9, 2 ** 9, (c,), generator=gen) * 2.0 ** -4).double()
    es = torch.randint(-3, 4, (c,), generator=gen)
    if far_pivot is None:
        far_pivot = torch.rand(c, generator=gen) < 0.5
    far_pivot = far_pivot & torch.tensor(n >= 8)
    x = torch.empty((n, c), dtype=torch.float64)
    sigma = torch.empty(c, dtype=torch.float64)
    for j in range(c):
        if bool(far_pivot[j]):
            m_out = 2 if k % 2 else 4                     # var = m_out A^2 / n: A = 2^a, 2a + log2(m_out) - k even
            a = int(es[j]) + (k - (1 if k % 2 else 2)) // 2
            A = 2.0 ** a
            col = torch.full((n,), float(mu[j]), dtype=torch.float64)
            idx = torch.cat([torch.zeros(1, dtype=torch.int64), 1 + torch.randperm(n - 1, generator=gen)[:m_out - 1]])
            signs = torch.tensor([1.0, -1.0, 1.0, -1.0][:m_out], dtype=torch.float64)
            col[idx] = mu[j] + signs * A
            x[:, j] = col
            sigma[j] = math.sqrt(m_out * A * A / n)
        else:
            s = 2.0 ** int(es[j])
            sg = torch.cat([torch.ones(n // 2), -torch.ones(n // 2)]).double()[torch.randperm(n, generator=gen)]
            x[:, j] = mu[j] + sg * s
            sigma[j] = s
    return x.float(), mu, sigma


def probe_affine(c, generator=None):
    """weights {0, +-1, +-2, +-3} 2^-2 (one zero channel), biases on the 2^-6 grid"""
    w = torch.tensor([1., -1., 2., -2., 3., -3.])[torch.randint(6, (c,), generator=generator)] * 0.25
    w[c // 2] = 0.0
    b = torch.randint(-64, 65, (c,), generator=generator).float() * 2.0 ** -6
    return w, b


def probe_grid_values(shape, lo_exp, hi_exp, generator=None):
    """fp32 values +-k 2^e, k in 0..3, e in [lo_exp, hi_exp]"""
    k = torch.randint(-3, 4, shape, generator=generator).float()
    e = torch.randint(lo_exp, hi_exp + 1, shape, generator=generator)
    return k * torch.exp2(e.float())


def exact_running(rm, rv, nbt, mu, sigma, n, momentum):
    """fp32 of the exact running-buffer update (Fraction arithmetic per channel): n / (n - 1) is not dyadic, so the
    exact value is never an fp32 tie and the kernel's fp64 evaluation must round to it"""
    tracked = int(nbt) + 1
    m = Fraction(1, tracked) if momentum is None else Fraction(momentum)
    out_m, out_v = [], []
    for j in range(rm.shape[0]):
        var = Fraction(float(sigma[j])) ** 2
        out_m.append(float((1 - m) * Fraction(float(rm[j])) + m * Fraction(float(mu[j]))))
        out_v.append(float((1 - m) * Fraction(float(rv[j])) + m * var * n / (n - 1)))
    f = lambda v: torch.tensor(v, dtype=torch.float64).float()
    return f(out_m), f(out_v), tracked


def budget_bits(terms_abs, grid):
    return R.exact_budget_bits(terms_abs, grid)


def exact_units(v, grid):
    """True where every value of v is a multiple of grid and below 2^24 grid (so fp32 holds it and sums of such values of
    magnitude < 2^24 grid are exact)"""
    q = v.double() / grid
    return bool(((q == torch.round(q)) & (q.abs() < 2.0 ** 24)).all())
