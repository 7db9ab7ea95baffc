"""NumPy restatement of the scene search contract (DESIGN.md, "Scene search contract"), given the fp16 score matrix.

Order: NaN never ranks, is never a maximum and is never counted; numbers by descending value with -0 == +0 and inf above
every finite value; equal values go to the lower global row.  ``rule`` selects deliberately wrong variants for the
negative controls of the CPU test: 'nan_first', 'tie_high', 'neg_zero_low', and 'boundary' (every scene offset but the
first and last moved up by one row)."""
import numpy as np

NEG_INF_BITS = np.uint16(0xfc00)


def order_keys(scores, rule=None):
    """int64 [N, nq] keys: larger is better, all distinct except -1 (NaN)."""
    s = np.ascontiguousarray(scores, dtype=np.float16)
    b = s.view(np.uint16).astype(np.int64)
    n = s.shape[0]
    u = np.where(b & 0x8000, (~b) & 0xffff, b | 0x8000)
    if rule != 'neg_zero_low':
        u = np.where(b == 0x8000, 0x8000, u)
    rows = np.arange(n, dtype=np.int64)[:, None]
    tie = rows if rule == 'tie_high' else 0xffffffff - rows
    key = (u << 32) | tie
    nan = np.isnan(s)
    if rule == 'nan_first':
        return np.where(nan, (np.int64(0x10000) << 32) | tie, key)
    return np.where(nan, -1, key)


def search_ref(scores, off, k, threshold=None, rule=None):
    """scores fp16 [N, nq], off int64 [S + 1] -> dict of score fp16 / scene / row [nq, k], scene_max fp16 /
    scene_argmax [S, nq], scene_count [S, nq] or None."""
    s = np.ascontiguousarray(scores, dtype=np.float16)
    off = np.asarray(off, dtype=np.int64)
    n, nq = s.shape
    if rule == 'boundary':
        off = off.copy()
        off[1:-1] += 1
    key = order_keys(s, rule)
    row_scene = np.repeat(np.arange(len(off) - 1), np.diff(off))
    score = np.full((nq, k), NEG_INF_BITS, np.uint16)
    scene = np.full((nq, k), -1, np.int64)
    row = np.full((nq, k), -1, np.int64)
    bits = s.view(np.uint16)
    for q in range(nq):
        kk = min(k, n)
        idx = np.argpartition(-key[:, q], kk - 1)[:kk]
        idx = idx[np.argsort(-key[idx, q], kind='stable')]
        idx = idx[key[idx, q] >= 0]
        m = len(idx)
        score[q, :m] = bits[idx, q]
        scene[q, :m] = row_scene[idx]
        row[q, :m] = idx - off[row_scene[idx]]
    kmax = np.maximum.reduceat(key, off[:-1], axis=0)                       # [S, nq]
    S = len(off) - 1
    scene_max = np.full((S, nq), NEG_INF_BITS, np.uint16)
    scene_arg = np.full((S, nq), -1, np.int64)
    has = kmax >= 0
    grow = 0xffffffff - (kmax & 0xffffffff) if rule != 'tie_high' else kmax & 0xffffffff
    if rule == 'nan_first':
        has = kmax >= 0
    cols = np.broadcast_to(np.arange(nq), (S, nq))
    scene_max[has] = bits[grow[has], cols[has]]
    scene_arg[has] = grow[has] - off[:-1, None].repeat(nq, 1)[has]
    count = None
    if threshold is not None:
        thr = np.broadcast_to(np.asarray(threshold, dtype=np.float32), (nq,))
        with np.errstate(invalid='ignore'):
            hit = (s.astype(np.float32) >= thr[None, :]).astype(np.int64)
        count = np.add.reduceat(hit, off[:-1], axis=0)
    return dict(score=score.view(np.float16), scene=scene, row=row, scene_max=scene_max.view(np.float16),
                scene_argmax=scene_arg, scene_count=count)
