"""NumPy restatement of the pooling contract (DESIGN.md "Pooling contract"), the yardstick of csrc/pool.cu.

Local pooling runs over an output-stationary map ``nbr[K][n_out]`` (input row feeding output o through offset k, -1 none):
  sum   fp32 adds over the present offsets in ascending k, from +0.0
  avg   fp32(sum) / fp32(max(count, 1))
  max   per channel the largest present input; the first NaN in offset order wins, ties (-0.0 == +0.0) go to the lowest k,
        an output with no present input gives 0 and winner NO_WINNER
  backward  gin[i] = fp32 adds in ascending k over the outputs o with nbr[k][o] = i of g[o] (sum), fp32(g[o] / count_o)
        (avg), g[o, c] where the winner of (o, c) is k (max; other outputs add nothing)
Global pooling reduces the rows of each batch index: sum / avg against fp64 with a per-element bound (the device sums
fp32 values in fp64 partials and rounds once), max exactly (first NaN, ties to the lowest row, empty batch -inf)."""
import numpy as np

SUM, AVG, MAX = 0, 1, 2
NO_WINNER = 0xFFFF


def pool_fwd(x, nbr, mode):
    """x float32 [n_in, C], nbr int [K, n_out] -> (out float32 [n_out, C], count int32 [n_out], winner uint16 [n_out, C])"""
    x = np.asarray(x, dtype=np.float32)
    nbr = np.asarray(nbr)
    K, n_out = nbr.shape
    acc = np.zeros((n_out, x.shape[1]), np.float32)
    win = np.full((n_out, x.shape[1]), NO_WINNER, np.uint16)
    cnt = np.zeros(n_out, np.int32)
    with np.errstate(invalid='ignore', over='ignore'):
        for k in range(K):
            o = np.nonzero(nbr[k] >= 0)[0]
            v = x[nbr[k][o]]
            cnt[o] += 1
            if mode == MAX:
                a, w = acc[o], win[o]
                take = (w == NO_WINNER) | (~np.isnan(a) & (np.isnan(v) | (v > a)))
                acc[o] = np.where(take, v, a)
                win[o] = np.where(take, np.uint16(k), w)
            else:
                acc[o] = acc[o] + v
        if mode == AVG:
            acc = acc / np.maximum(cnt, 1).astype(np.float32)[:, None]
    return acc, cnt, win


def pool_bwd(g, nbr, mode, count, win, n_in):
    """g float32 [n_out, C] over the forward map nbr [K, n_out] -> gin float32 [n_in, C]"""
    g = np.asarray(g, dtype=np.float32)
    nbr = np.asarray(nbr)
    gin = np.zeros((n_in, g.shape[1]), np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        for k in range(nbr.shape[0]):
            o = np.nonzero(nbr[k] >= 0)[0]
            i = nbr[k][o]                                   # one input per (k, o) and one output per (k, i)
            if mode == SUM:
                gin[i] = gin[i] + g[o]
            elif mode == AVG:
                gin[i] = gin[i] + g[o] / np.maximum(count[o], 1).astype(np.float32)[:, None]
            else:
                gin[i] = np.where(win[o] == k, gin[i] + g[o], gin[i])
    return gin


def transpose_map(nbr, n_in):
    """nbr [K, n_out] -> nbr_t [K, n_in] (output row per (k, input row), -1 none)"""
    nbr = np.asarray(nbr)
    t = np.full((nbr.shape[0], n_in), -1, np.int32)
    for k in range(nbr.shape[0]):
        o = np.nonzero(nbr[k] >= 0)[0]
        t[k, nbr[k][o]] = o
    return t


def global_sum64(x, batch, n_batch):
    """(fp64 sums [B, C], sums of |x| [B, C], row counts [B]) -- exact for dyadic inputs of a bounded range"""
    x = np.asarray(x, dtype=np.float64)
    s = np.zeros((n_batch, x.shape[1]))
    a = np.zeros((n_batch, x.shape[1]))
    np.add.at(s, batch, x)
    np.add.at(a, batch, np.abs(x))
    return s, a, np.bincount(batch, minlength=n_batch)


def global_fwd_exact(x, batch, n_batch, mode):
    """the device result when every fp64 partial sum is exact (dyadic probes); max is exact for any input.
    -> (out float32 [B, C], count int32 [B], argrow int32 [B, C])"""
    x = np.asarray(x, dtype=np.float32)
    batch = np.asarray(batch)
    c = x.shape[1]
    argrow = np.full((n_batch, c), -1, np.int32)
    if mode == MAX:
        out = np.full((n_batch, c), -np.inf, np.float32)
        for b in range(n_batch):
            rows = np.nonzero(batch == b)[0]
            if not len(rows):
                continue
            v = x[rows]
            nan = np.isnan(v)
            with np.errstate(invalid='ignore'):
                first = np.where(nan.any(0), nan.argmax(0), np.where(nan, -np.inf, v).argmax(0))
            argrow[b] = rows[first]
            out[b] = v[first, np.arange(c)]
        return out, np.bincount(batch, minlength=n_batch).astype(np.int32), argrow
    s, _, n = global_sum64(x, batch, n_batch)
    if mode == AVG:
        with np.errstate(invalid='ignore', divide='ignore'):
            s = s / n[:, None]
    return s.astype(np.float32), n.astype(np.int32), argrow


def global_sum_bound(x, batch, n_batch, mode):
    """(fp64 reference [B, C], per-element bound) for the device's fp64-partial sums of arbitrary fp32 inputs: each partial
    and merge add is an fp64 rounding (<= n_b adds of relative 2^-53 against sum |x|), the average one more fp64 division,
    then one rounding to fp32 (half an fp32 spacing of the value reached)"""
    s, a, n = global_sum64(x, batch, n_batch)
    d = (n[:, None] + 2) * 2.0 ** -52 * a
    ref = s
    if mode == AVG:
        with np.errstate(invalid='ignore', divide='ignore'):
            ref, d = s / n[:, None], d / np.maximum(n, 1)[:, None] + 2.0 ** -52 * np.abs(s / np.maximum(n, 1)[:, None])
    spacing = np.spacing(np.abs(ref + d).astype(np.float32)).astype(np.float64)
    return ref, d + 0.5 * spacing + 1e-45


def global_bwd(g, batch, mode, count, argrow):
    """gin [n, C]: g[b] (sum), fp32(g[b] / count_b) (avg), g[b, c] on the winning row and 0 elsewhere (max)"""
    g = np.asarray(g, dtype=np.float32)
    batch = np.asarray(batch)
    gb = g[batch]
    if mode == SUM:
        return gb.copy()
    if mode == AVG:
        return gb / count[batch].astype(np.float32)[:, None]
    rows = np.arange(len(batch))[:, None]
    return np.where(argrow[batch] == rows, gb, np.float32(0))
