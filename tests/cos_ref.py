"""fp64 restatement of run/distill.py's cosine loss, ``(1 - torch.nn.CosineSimilarity(dim=1, eps=1e-8)(f, t)).mean()``, as
torch 2.11 computes it, and the closed-form gradient the device head (csrc/cos_head.cu) implements:

    n1 = |f|, n2 = |t|, n1c = max(n1, eps), n2c = max(n2, eps)    (the clamps under no_grad)
    cos = sum_j (f_j / n1c) (t_j / n2c)
    dloss/df_r = a_r t_r + b_r f_r,  a_r = -g / (M n1c n2c),  b_r = g (f.t) / (M n1c^2 n2c n1)  (b_r = 0 when n1 = 0)

``head`` is the fp64 reference of the two head launches (osb_cos_head_fwd / osb_cos_head_bwd) on the operands they read, with
per-element bounds, shared by tests/test_gpu_cos_head.py (the kernels alone) and tests/test_gpu_norm_replay.py (every launch
of the engine's cosine step).  Bounds, u = 2^-24, g_k = k u / (1 - k u), E = g_cin |X| |W| the error bound of the fp32 products
f = x W:
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
         s = rows per split = ceil(m / min(ceil(m / 512), 64))  (``dw_split_rows``)
Every bound gets a factor 1.5 for the second-order terms dropped above."""
import math

import torch

EPS = 1e-8
U = 2.0 ** -24
DW_SPLIT_ROWS, DW_MAX_SPLITS = 512, 64            # csrc/cos_head.cu: cos_splits
SPLIT_STORE = 2.0 ** -17
SLACK = 1.5


def cos_loss(f, t, eps=EPS):
    """the loss, with autograd, through the operations of torch's cosine_similarity"""
    n1 = torch.linalg.vector_norm(f, 2, dim=-1, keepdim=True)
    n2 = torch.linalg.vector_norm(t, 2, dim=-1, keepdim=True)
    # the clamp without gradient: the value of max(n, eps), the derivative of n
    n1 = n1 + (n1.detach().clamp_min(eps) - n1.detach())
    n2 = n2 + (n2.detach().clamp_min(eps) - n2.detach())
    return (1 - ((f / n1) * (t / n2)).sum(1)).mean()


def cos_ab(n1, ft, n2, m, g=1.0, eps=EPS):
    """(a, b) per row from |f|, f.t, |t| (fp64 tensors), the scalars of dloss/df = a t + b f"""
    n1c, n2c = n1.clamp_min(eps), n2.clamp_min(eps)
    a = -g / (m * n1c * n2c)
    b = torch.where(n1 > 0, g * ft / (m * n1c * n1c * n2c * n1.clamp_min(1e-300)), torch.zeros_like(n1))
    return a, b


def cos_grad(f, t, g=1.0, eps=EPS):
    """closed-form dloss/df"""
    n1, n2, ft = f.norm(dim=1), t.norm(dim=1), (f * t).sum(1)
    a, b = cos_ab(n1, ft, n2, f.shape[0], g, eps)
    return a[:, None] * t + b[:, None] * f


def gam(k):
    return k * U / (1 - k * U)


def dw_splits(m):
    return min(math.ceil(m / DW_SPLIT_ROWS), DW_MAX_SPLITS)


def dw_split_rows(m):
    """rows per split of the dW partials"""
    return math.ceil(m / dw_splits(m))


def head(x, w, t, rows, g=1.0):
    """fp64 reference and per-element bound of both head launches.  x: fp64 [n, cin] every row as the head reads it (split
    rows joined, e.g. ``replay_ref.split_decode``), w: [cin, C], t: the fp16 targets widened, [m, C] in the order of rows
    (int, internal row of each supervised row), g: the upstream gradient.  Returns {name: (reference, bound)} for
    'state' [m, 3] (|f|, f.t, |t|), 'loss' (0-dim), 'dx' [m, cin] (the supervised rows, in the order of rows) and 'dW'
    [cin, C]; an output is within its bound when |got - reference| <= bound element by element."""
    r = rows.long()
    m, cin = r.shape[0], x.shape[1]
    c = w.shape[1]
    X, W, T = x.double()[r], w.double(), t.double()
    F = X @ W
    n1, n2, ft = F.norm(dim=1), T.norm(dim=1), (F * T).sum(1)
    n1c, n2c = n1.clamp_min(EPS), n2.clamp_min(EPS)
    cos = ft / (n1c * n2c)
    loss = (1 - cos).mean()
    E = gam(cin) * (X.abs() @ W.abs())
    dn1 = E.norm(dim=1)
    dft = (E * T.abs()).sum(1)
    state = torch.stack([n1, ft, n2], 1)
    state_b = torch.stack([SLACK * dn1 + 1e-12 * n1, SLACK * dft + 1e-12 * (F * T).abs().sum(1), 1e-12 * n2], 1)
    loss_b = ((dft / (n1c * n2c) + cos.abs() * dn1 / n1c).sum() / m + U * loss.abs()) * SLACK

    a, b = cos_ab(n1, ft, n2, m, g)
    n1s = n1.clamp_min(1e-300)
    da = a.abs() * (dn1 / n1c + U)
    db = torch.where(n1 > 0, b.abs() * (3 * dn1 / n1s + U) + abs(g) * dft / (m * n1c * n1c * n2c * n1s), torch.zeros_like(n1))
    P, Q = T @ W.t(), F @ W.t()
    G = W @ W.t()
    dx = a[:, None] * P + b[:, None] * Q
    dx_b = (da[:, None] * P.abs() + a.abs()[:, None] * gam(c) * (T.abs() @ W.abs().t())
            + db[:, None] * Q.abs() + b.abs()[:, None] * (gam(cin) * (X.abs() @ G.abs()) + gam(c) * (X.abs() @ (W.abs() @ W.abs().t())))
            + U * (a.abs()[:, None] * P.abs() + 2 * b.abs()[:, None] * Q.abs()) + SPLIT_STORE * dx.abs()) * SLACK
    gs = gam(dw_split_rows(m) + 1)
    dW = X.t() @ (a[:, None] * T) + (X.t() @ (b[:, None] * X)) @ W
    dW_b = ((X.abs().t() @ ((da + gs * a.abs())[:, None] * T.abs()))
            + (X.abs().t() @ ((db + gs * b.abs())[:, None] * X.abs())) @ W.abs() + U * dW.abs()) * SLACK
    return dict(state=(state, state_b), loss=(loss, loss_b), dx=(dx, dx_b), dW=(dW, dW_b))


def ratio(got, ref, bound):
    """max over elements of |got - ref| / bound (0 where both are 0; inf where the bound is 0 and the error is not)"""
    err = (got.double() - ref).abs()
    r = err / bound
    r = torch.where(err == 0, torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def ratios(got, ref):
    """{name: ratio} of the outputs in got ({name: tensor}) against head()'s {name: (reference, bound)}"""
    return {k: ratio(v, *ref[k]) for k, v in got.items()}


def case(m, cin, c, seed, edges=False):
    """(x fp32 [n, cin], w fp32 [cin, C], rows int32 [m], t fp16 [m, C]) on the CPU, n = m + m // 2 + 7 (unsupervised rows
    too).  edges: supervised row 1 has x = 0 (a zero output row), row 2 one channel of 1e-10 (0 < |f| < eps without
    cancellation in x W), row 3 a zero target (dx exactly 0)."""
    g = torch.Generator().manual_seed(seed)
    n = m + m // 2 + 7
    x = torch.randn(n, cin, generator=g)
    w = torch.randn(cin, c, generator=g) / cin ** 0.5
    rows = torch.randperm(n, generator=g)[:m].to(torch.int32)
    t = torch.randn(m, c, generator=g).half()
    if edges:
        r = rows.long()
        x[r[1]] = 0
        x[r[2]] = 0
        x[r[2], 5] = 1e-10
        t[3] = 0
    return x, w, rows, t


def edge_rows(c, dtype=torch.float64, seed=0):
    """(f, t): random rows plus a zero output row, a row with 0 < |f| < eps, a zero target row and a NaN row (last)"""
    gen = torch.Generator().manual_seed(seed)
    f = torch.randn(8, c, generator=gen, dtype=dtype)
    t = torch.randn(8, c, generator=gen, dtype=dtype)
    f[1] = 0
    f[2] = f[2] / f[2].norm() * 3e-9
    t[3] = 0
    f[7, 5] = float('nan')
    return f, t
