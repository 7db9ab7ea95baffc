"""NumPy restatement of csrc/optim.cu's updates, rounding for rounding (fp32, FMAs included), and their fp64 error bounds.

``fma32(a, b, c)`` is fp32 ``fma`` with one rounding: ``a * b`` is exact in fp64, ``a * b + c`` is carried as an fp64 sum plus
its exact error (TwoSum), and the fp64 sum's rounding to fp32 is corrected where it lands exactly on a tie that the error
breaks."""
import numpy as np

F32 = np.float32
U = 2.0 ** -24                 # unit roundoff of fp32
TINY = 2.0 ** -148             # two subnormal ulps: the absolute floor of every bound


def fma32(a, b, c):
    a, b, c = (np.asarray(x, dtype=np.float64) for x in (a, b, c))
    with np.errstate(all='ignore'):
        p = a * b
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        r = s.astype(np.float32)
        d = s - r.astype(np.float64)
        nxt = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf))).astype(np.float64)
        tie = np.isfinite(s) & (d != 0) & (nxt - s == d) & (err != 0)
        up = tie & (np.sign(err) == np.sign(d))
        r = np.where(up, nxt.astype(np.float32), r)
    return r.astype(np.float32)


def lerp(m, g, w):
    """torch's lerp (ATen/native/Lerp.h) as its CUDA build contracts it"""
    w = F32(w)
    with np.errstate(all='ignore'):
        d = (g - m).astype(np.float32)
        if abs(w) < 0.5:
            return fma32(w, d, m)
        return fma32(-d, F32(1) - w, g)


def adam(p, g, m, v, step_size, bc2_sqrt, lerp_w, beta2, one_minus_beta2, eps):
    """-> (p, m, v) of one osb_optim_adam element-wise update (all fp32 arrays / scalars)"""
    with np.errstate(all='ignore'):
        m = lerp(m, g, lerp_w)
        v = fma32(F32(one_minus_beta2), (g * g).astype(np.float32), (v * F32(beta2)).astype(np.float32))
        denom = (np.sqrt(v) / F32(bc2_sqrt)).astype(np.float32) + F32(eps)
        p = fma32(F32(step_size), (m / denom).astype(np.float32), p)
    return p, m, v


def sgd(p, g, buf, neg_lr, weight_decay, momentum, first):
    """-> (p, buf) of one osb_optim_sgd update; buf None: no momentum"""
    with np.errstate(all='ignore'):
        d = fma32(F32(weight_decay), p, g) if weight_decay != 0 else g.astype(np.float32)
        if buf is not None:
            d = d if first else ((buf * F32(momentum)).astype(np.float32) + d).astype(np.float32)
            buf = d
        p = fma32(F32(neg_lr), d, p)
    return p, buf


def adam_bound(p, g, m, v, step_size, bc2_sqrt, lerp_w, beta2, one_minus_beta2, eps):
    """(fp64 result, per-element bound on |fp32 result - fp64 result|) of the new parameter, from the same fp32 inputs;
    no bound (inf) where the fp32 arithmetic overflows"""
    p, g, m, v = (np.asarray(x, dtype=np.float64) for x in (p, g, m, v))
    ss, bc2, w, b2, s2, eps = (float(F32(x)) for x in (step_size, bc2_sqrt, lerp_w, beta2, one_minus_beta2, eps))
    with np.errstate(all='ignore'):
        m1 = m + w * (g - m)
        v1 = v * b2 + s2 * g * g
        den = np.sqrt(v1) / bc2 + eps
        q = m1 / den
        p1 = p + ss * q
        e_m = U * (np.abs(m1) + abs(w) * np.abs(g - m) + np.abs(g) + np.abs(m))
        bound = 2 * (U * np.abs(p1) + abs(ss) * (e_m + 10 * U * np.abs(m1)) / den) + TINY
        # where g * g overflows fp32 (|g| > 1.8e19) v becomes inf and the fp32 update 0, in torch as here: no fp64 bound
        g32 = g.astype(np.float32)
        bound = np.where(np.isfinite(g32) & ~np.isfinite(g32 * g32), np.inf, bound)
    return p1, bound


def sgd_bound(p, g, buf, neg_lr, weight_decay, momentum, first):
    p, g = np.asarray(p, dtype=np.float64), np.asarray(g, dtype=np.float64)
    lr, wd, mu = (float(F32(x)) for x in (neg_lr, weight_decay, momentum))
    with np.errstate(all='ignore'):
        d = g + wd * p
        mag = np.abs(g) + np.abs(wd * p)
        if buf is not None:
            b = np.asarray(buf, dtype=np.float64)
            d = d if first else b * mu + d
            mag = mag + (0 if first else np.abs(b * mu))
        p1 = p + lr * d
        bound = 4 * U * (np.abs(p1) + abs(lr) * (np.abs(d) + mag)) + TINY
    return p1, bound
