"""fp64 restatement of run/distill.py's cosine loss, ``(1 - torch.nn.CosineSimilarity(dim=1, eps=1e-8)(f, t)).mean()``, as
torch 2.11 computes it, and the closed-form gradient the device head (csrc/cos_head.cu) implements:

    n1 = |f|, n2 = |t|, n1c = max(n1, eps), n2c = max(n2, eps)    (the clamps under no_grad)
    cos = sum_j (f_j / n1c) (t_j / n2c)
    dloss/df_r = a_r t_r + b_r f_r,  a_r = -g / (M n1c n2c),  b_r = g (f.t) / (M n1c^2 n2c n1)  (b_r = 0 when n1 = 0)"""
import torch

EPS = 1e-8


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
