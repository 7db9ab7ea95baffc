"""NumPy restatement of the label contract (DESIGN.md, "Label contract"), given the fp16 score matrix of the index's rows
against the vocabulary.

* label: per row the first NaN column, else the first maximum with -0 == +0 (``osb_match_topk`` with topk = 1), and its
  fp16 score;
* class matrix T [N, m]: T[r, j] = the label score of r when its label is classes[j], else NaN;
* class counts: without a threshold every row under its label (NaN scores included); with one, ``search_ref``'s
  ``scene_count`` of T;
* class regions: ``regions_ref`` of T with the thresholds (default -inf).

``rule`` selects deliberately wrong variants for the negative controls of the CPU test: 'tie_high' (ties to the higher
column), 'second_best' (the slot taken from the row's second-best label), 'nan_hit' (a NaN score counted under a
threshold), 'merge_classes' (the hits of every listed class grown together) and 'cross_scene' (regions across scenes)."""
import numpy as np

from tests.regions_ref import regions_ref
from tests.search_ref import search_ref


def label_ref(scores, rule=None):
    """scores fp16 [N, K] -> (label int64 [N], score fp16 [N])"""
    s = np.ascontiguousarray(scores, dtype=np.float16)
    n, K = s.shape
    v = s.astype(np.float64)
    nan = np.isnan(v)
    vv = np.where(nan, -np.inf, v)
    if rule == 'second_best':
        order = np.lexsort((np.broadcast_to(np.arange(K), (n, K)), -vv, ~nan), axis=-1)
        lab = order[:, min(1, K - 1)]
    else:
        best = (vv == vv.max(1, keepdims=True))
        if rule == 'tie_high':
            first = K - 1 - best[:, ::-1].argmax(1)
        else:
            first = best.argmax(1)
        lab = np.where(nan.any(1), nan.argmax(1), first)
    lab = lab.astype(np.int64)
    return lab, s[np.arange(n), lab]


def class_matrix(label, score, classes, rule=None):
    """T fp16 [N, m]"""
    label = np.asarray(label, np.int64)
    score = np.asarray(score, np.float16)
    cls = np.asarray(classes, np.int64)
    mine = label[:, None] == cls[None, :]
    if rule == 'merge_classes':
        mine = np.broadcast_to(np.isin(label, cls)[:, None], mine.shape)
    return np.where(mine, score[:, None], np.float16(np.nan)).astype(np.float16)


def class_counts_ref(label, score, off, classes, threshold=None, rule=None):
    """int64 [S, m]"""
    T = class_matrix(label, score, classes)
    m = T.shape[1]
    if threshold is None:
        hit = (np.asarray(label)[:, None] == np.asarray(classes)[None, :]).astype(np.int64)
        return np.add.reduceat(hit, np.asarray(off)[:-1], axis=0)
    thr = np.broadcast_to(np.asarray(threshold, np.float32), (m,))
    if rule == 'nan_hit':
        with np.errstate(invalid='ignore'):
            hit = (T.astype(np.float32) >= thr) | (np.isnan(T) & (np.asarray(label)[:, None] == np.asarray(classes)))
        return np.add.reduceat(hit.astype(np.int64), np.asarray(off)[:-1], axis=0)
    return search_ref(T, off, 1, threshold=thr)['scene_count']


def class_regions_ref(label, score, coords, off, classes, threshold=None, R=8, reach=1, min_voxels=1, rule=None):
    """the regions_ref dict of T"""
    T = class_matrix(label, score, classes, rule)
    m = T.shape[1]
    thr = np.full(m, -np.inf, np.float32) if threshold is None else \
        np.broadcast_to(np.asarray(threshold, np.float32), (m,))
    return regions_ref(T, coords, off, thr, R, reach, min_voxels, rule='cross_scene' if rule == 'cross_scene' else None)
