"""The ordering rule of the streaming top-k match (osb_match_topk, osb_match_ensemble_topk; DESIGN.md "Top-k match contract"),
restated in NumPy, with a torch version for GPU-sized inputs that tests/test_match_topk_cpu.py checks against it.

Per row of fp16 scores, the k best columns, best first:
* every NaN ranks above every number, NaNs by ascending column;
* numbers rank by descending value, -0 equal to +0 (inf above every finite value);
* equal values go to the lower column.
For k = 1 this is the argmax of tests/vote_oracle.py (torch's CPU ``x.float().max(1)[1]``)."""
import numpy as np
import torch


def topk(s, k, cols=None):
    """(labels int64 [n, k], scores fp16 [n, k]) of the fp16 scores s [n, K] (numpy); cols [n, K] gives each score's column
    (default: its position), so that per-slice results can be merged by calling topk again on their concatenation"""
    s = np.asarray(s, dtype=np.float16)
    n, K = s.shape
    if not 1 <= k <= K:
        raise ValueError(f"topk: k={k} outside 1..K={K}")
    cols = np.broadcast_to(np.arange(K, dtype=np.int64), s.shape) if cols is None else np.asarray(cols, dtype=np.int64)
    v = s.astype(np.float64)
    nan = np.isnan(v)
    val = np.where(nan, 0.0, v) + 0.0                 # -0 + 0 = +0
    # np.lexsort: the last key is the primary one; numbers compare by value, so equal values fall through to the column
    order = np.lexsort((cols, -val, ~nan), axis=-1)[:, :k]
    return np.take_along_axis(cols, order, 1), np.take_along_axis(s, order, 1)


def topk_torch(s, k, cols=None):
    """topk on torch tensors (any device): three stable sorts, least significant key first"""
    n, K = s.shape
    if not 1 <= k <= K:
        raise ValueError(f"topk: k={k} outside 1..K={K}")
    cols = torch.arange(K, device=s.device).expand(n, K) if cols is None else cols
    order = torch.sort(cols, dim=1, stable=True).indices
    v = s.float().gather(1, order)
    nan = torch.isnan(v)
    val = torch.where(nan, torch.zeros_like(v), v) + 0.0
    order = order.gather(1, torch.sort(-val, dim=1, stable=True).indices)
    order = order.gather(1, torch.sort((~torch.isnan(s.float().gather(1, order))).to(torch.uint8), dim=1,
                                       stable=True).indices)[:, :k]
    return cols.gather(1, order), s.gather(1, order)
