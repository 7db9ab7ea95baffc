"""fp64 restatement of run/distill.py's L1 loss, ``torch.nn.L1Loss()(f, t)`` = ``abs(f - t).mean()``, as torch 2.11 computes it,
and of the device head (csrc/l1_head.cu) that implements it:

    d = fp32(f - t)                     f = x W in fp32, t the fp16 target widened exactly
    loss = sum |d| / (M C)
    dloss/df = s sgn(d),  sgn(d) = (0 < d) - (d < 0)   (0 at d = +-0 and at NaN)
    s = fp32(g * fp32(1 / fp32(M C)))   torch's CUDA MeanBackward0: a tensor divided by a CPU scalar is multiplied by the
                                        fp32 reciprocal (``scale``; tests/test_gpu_l1_head.py checks it against torch)
    dx_r = s (sgn_r W^T),  dW = s (X^T Sgn)

The forward keeps sgn(d) as 2-bit codes, uint32 [M, C / 16] (``pack`` / ``decode``): element j of a row is bits
2 (j % 16) .. 2 (j % 16) + 1 of word j / 16, code 0 for sign 0, 1 for +1, 2 for -1.

``head`` is the fp64 reference of the two head launches (osb_l1_head_fwd / osb_l1_head_bwd) on the operands they read, with
per-element bounds, shared by tests/test_gpu_l1_head.py (the kernels alone) and tests/test_gpu_l1_replay.py (the launches of
the engine's L1 step).  Bounds, u = 2^-24, g_k = k u / (1 - k u), E = g_cin |X| |W| the error bound of the fp32 products:
  d      |d dev - d| <= E + u |d|; a stored sign must equal sign(d) wherever |d| exceeds that bound
  loss   <= (sum (E + u |d|) / (M C)) + u |loss|  (the fp64 sum and division are exact to far below that)
  dx_rk  from the stored signs S (exact +-1 / 0): s g_C (|S| |W|^T) + u |dx| (the product by s) + 2^-17 |dx| (split store)
  dW_kj  s g_{rows per split + 1} (|X|^T |S|) + u |dW|  (fp32 within a split, splits merged in fp64, one rounding of s sum)
Every bound gets a factor 1.5 for the second-order terms dropped above."""
import math

import numpy as np
import torch

U = 2.0 ** -24
DW_SPLIT_ROWS, DW_MAX_SPLITS = 512, 64            # csrc/l1_head.cu: l1_splits
SPLIT_STORE = 2.0 ** -17
SLACK = 1.5


def l1_loss(f, t):
    """the loss as run/distill.py computes it (``distill.distill_loss(f, t, 'l1')``), with autograd"""
    return torch.nn.L1Loss()(f, t.to(f.dtype))


def scale(g, m, c):
    """s: the fp32 value of g / (M C) that torch's CUDA MeanBackward0 gives every element"""
    inv = np.float32(1.0) / np.float32(m * c)
    return float(np.float32(g) * inv)


def sgn(d):
    """torch's sgn: (0 < d) - (d < 0), int8; NaN and +-0 give 0"""
    return ((d > 0).to(torch.int8) - (d < 0).to(torch.int8))


def pack(s):
    """int8 signs [M, C] -> int32 code words [M, C / 16] (the bits of the uint32 words the kernel writes)"""
    m, c = s.shape
    code = torch.where(s > 0, 1, torch.where(s < 0, 2, 0)).to(torch.int64).reshape(m, c // 16, 16)
    words = (code << (2 * torch.arange(16, dtype=torch.int64))).sum(2)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def decode(words, c, strict=True):
    """int32 / uint32 code words [M, C / 16] -> int8 signs [M, C]; strict: code 3 (never written) raises"""
    w = words.cpu().to(torch.int64) & 0xFFFFFFFF
    code = (w[:, :, None] >> (2 * torch.arange(16, dtype=torch.int64))) & 3
    if strict and bool((code == 3).any()):
        raise AssertionError("sign code 3 written")
    code = code.reshape(w.shape[0], c)
    return (code == 1).to(torch.int8) - (code == 2).to(torch.int8)


def gam(k):
    return k * U / (1 - k * U)


def dw_splits(m):
    return min(math.ceil(m / DW_SPLIT_ROWS), DW_MAX_SPLITS)


def dw_split_rows(m):
    """rows per split of the dW partials"""
    return math.ceil(m / dw_splits(m))


def head(x, w, t, rows, signs=None, g=1.0, s=None):
    """fp64 reference and per-element bound of both head launches.  x: fp64 [n, cin] every row as the head reads it (split
    rows joined), w: [cin, C], t: the fp16 targets widened, [m, C] in the order of rows (int, internal row of each supervised
    row), signs: the int8 signs the backward reads ([m, C], the forward's stored signs decoded; None: the fp64 signs of d),
    g: the upstream gradient, s: a scale in place of ``scale(g, M, C)`` (negative controls).  Returns {name: (reference,
    bound)} for 'd' [m, C] (the bound decides where a stored sign is certain), 'loss' (0-dim), 'dx' [m, cin] (the supervised
    rows, in the order of rows) and 'dW' [cin, C]."""
    r = rows.long().cpu()
    m, cin = r.shape[0], x.shape[1]
    c = w.shape[1]
    X, W, T = x.double().cpu()[r], w.double().cpu(), t.double().cpu()
    F = X @ W
    D = F - T
    E = gam(cin) * (X.abs() @ W.abs())
    d_b = SLACK * (E + U * D.abs())
    loss = D.abs().sum() / (m * c)
    loss_b = SLACK * ((E + U * D.abs()).sum() / (m * c) + U * loss.abs())
    S = (sgn(D) if signs is None else signs.cpu()).double()
    s = scale(g, m, c) if s is None else s
    P = S @ W.t()
    dx = s * P
    dx_b = SLACK * (abs(s) * gam(c) * (S.abs() @ W.abs().t()) + (U + SPLIT_STORE) * dx.abs())
    dW = s * (X.t() @ S)
    dW_b = SLACK * (abs(s) * gam(dw_split_rows(m) + 1) * (X.abs().t() @ S.abs()) + U * dW.abs())
    return dict(d=(D, d_b), loss=(loss, loss_b), dx=(dx, dx_b), dW=(dW, dW_b))


def certain(ref):
    """bool [m, C]: the elements whose sign the forward bound decides"""
    D, b = ref['d']
    return D.abs() > b


def ratio(got, ref, bound):
    """max over elements of |got - ref| / bound (0 where both are equal; inf where the bound is 0 and the error is not)"""
    got, ref = got.double().cpu(), ref.double()
    err = (got - ref).abs()
    r = err / bound
    r = torch.where((err == 0) | (got == ref), torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def ratios(got, ref):
    """{name: ratio} of the outputs in got ({name: tensor}) against head()'s {name: (reference, bound)}"""
    return {k: ratio(v, *ref[k]) for k, v in got.items()}


def emulate(x, w, t, rows, g=1.0):
    """fp32 CPU emulation of the documented kernel arithmetic: (loss, int8 signs, dx [m, cin] of the supervised rows after the
    split store, dW)"""
    r = rows.long()
    m, cin = r.shape[0], x.shape[1]
    c = w.shape[1]
    X, W, T = x.float()[r], w.float(), t.float()
    f = torch.zeros(m, c)
    for k in range(cin):                                  # k ascending, one rounding per step
        f = f + X[:, k:k + 1] * W[k]
    d = f - T
    loss = torch.tensor(float(d.double().abs().sum() / (m * c)), dtype=torch.float32)
    S = sgn(d)
    s = torch.tensor(scale(g, m, c), dtype=torch.float32)
    Sf = S.float()
    p = torch.zeros(m, cin)
    for j in range(c):                                    # j ascending
        p = p + Sf[:, j:j + 1] * W[:, j]
    v = s * p
    hi = v.bfloat16().float()
    dx = hi + (v - hi).bfloat16().float()
    acc = torch.zeros(cin, c, dtype=torch.float64)
    rps = dw_split_rows(m)
    for r0 in range(0, m, rps):
        part = torch.zeros(cin, c)
        for i in range(r0, min(m, r0 + rps)):            # rows ascending in fp32
            part = part + X[i][:, None] * Sf[i][None, :]
        acc = acc + part.double()
    dW = (float(s) * acc).float()
    return loss, S, dx, dW


def case(m, cin, c, seed):
    """(x fp32 [n, cin], w fp32 [cin, C], rows int32 [m], t fp16 [m, C]) on the CPU, n = m + m // 2 + 7 (unsupervised rows
    too); t is f plus noise, so signs of both kinds and small |d| occur"""
    g = torch.Generator().manual_seed(seed)
    n = m + m // 2 + 7
    x = torch.randn(n, cin, generator=g)
    w = torch.randn(cin, c, generator=g) / cin ** 0.5
    rows = torch.randperm(n, generator=g)[:m].to(torch.int32)
    t = (x[rows.long()] @ w + 0.5 * torch.randn(m, c, generator=g)).half()
    return x, w, rows, t


def exact_case(m, cin, c, seed):
    """dyadic operands with exact products: x in multiples of 1/4 up to 2, w in multiples of 1/8 up to 1, with at most 12
    nonzero channels per row of x, so f = x W is exact in fp32 whatever the order; t = f rounded to fp16 (ties where f is an
    fp16 value) with planted edges: row 0 t = f exactly (every d = +-0 or 0), t[1, 0:3] = NaN, +inf, -inf, and in row 2
    alternate columns of t = -0 against f = 0 (x row 2 is zero)."""
    g = torch.Generator().manual_seed(seed)
    n = m + 5
    x = torch.randint(-8, 9, (n, cin), generator=g).float() / 4
    keep = torch.rand(n, cin, generator=g) < 12 / cin
    x = x * keep
    w = torch.randint(-8, 9, (cin, c), generator=g).float() / 8
    rows = torch.randperm(n, generator=g)[:m].to(torch.int32)
    r = rows.long()
    if m > 2:
        x[r[2]] = 0
    f = x[r] @ w
    t = (f + torch.randint(-2, 3, (m, c), generator=g).float() / 4).half()
    t[0] = f[0].half()
    if m > 1:
        t[1, 0], t[1, 1], t[1, 2] = float('nan'), float('inf'), float('-inf')
    if m > 2:
        t[2, ::2] = -0.0
    return x, w, rows, t
