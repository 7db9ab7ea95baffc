"""NumPy / SciPy restatement of the region contract (DESIGN.md, "Region contract"), given the fp16 score matrix, the voxel
coordinates and the scene offsets.

A hit is (r, q) with float(s[r, q]) >= thr[q] (NaN never).  Hits of one query in one scene are adjacent at Chebyshev
distance <= reach; regions are the connected components (``cKDTree.query_pairs(p=inf)`` and
``scipy.sparse.csgraph.connected_components``, not the device's union-find).  Per query the regions of at least
``min_voxels`` voxels rank by the search order of their best hit (``search_ref.order_keys``).  ``rule`` selects
deliberately wrong variants for the negative controls: 'six' (6-connectivity), 'by_size' (rank by size, then best key),
'tie_high' (ties to the higher row), 'nan_hit' (NaN counted as a hit at the top of the order) and 'cross_scene' (regions
may cross a scene boundary)."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

from tests.search_ref import NEG_INF_BITS, order_keys


def _components(xyz, reach, rule):
    n = len(xyz)
    if n == 1:
        return np.zeros(1, np.int64)
    pairs = cKDTree(xyz.astype(np.float64)).query_pairs(r=reach + 0.5 if rule != 'six' else 1.0,
                                                         p=np.inf if rule != 'six' else 1, output_type='ndarray')
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(n, n))
    return connected_components(g, directed=False)[1]


def regions_ref(scores, coords, off, threshold, R, reach=1, min_voxels=1, rule=None):
    """scores fp16 [N, nq], coords int [N, 3], off [S + 1], threshold [nq] -> dict of score fp16 / scene / row / size
    [nq, R], box_min / box_max int32 [nq, R, 3], n_regions [S, nq], and the hit list (hit_query, hit_scene, hit_row,
    hit_score, hit_region) sorted by (query, global row)."""
    s = np.ascontiguousarray(scores, dtype=np.float16)
    xyz = np.asarray(coords, dtype=np.int64)[:, :3]
    off = np.asarray(off, dtype=np.int64)
    n, nq = s.shape
    S = len(off) - 1
    thr = np.broadcast_to(np.asarray(threshold, dtype=np.float32), (nq,))
    key = order_keys(s, 'tie_high' if rule == 'tie_high' else None)
    row_scene = np.repeat(np.arange(S), np.diff(off))
    with np.errstate(invalid='ignore'):
        hit = s.astype(np.float32) >= thr[None, :]
    if rule == 'nan_hit':
        hit |= np.isnan(s)
        key = np.where(np.isnan(s), (np.int64(0x10000) << 32) | (0xffffffff - np.arange(n)[:, None]), key)
    bits = s.view(np.uint16)
    out = dict(score=np.full((nq, R), NEG_INF_BITS, np.uint16), scene=np.full((nq, R), -1, np.int64),
               row=np.full((nq, R), -1, np.int64), size=np.zeros((nq, R), np.int64),
               box_min=np.zeros((nq, R, 3), np.int32), box_max=np.zeros((nq, R, 3), np.int32),
               n_regions=np.zeros((S, nq), np.int64))
    hq, hr, hreg = [], [], []
    for q in range(nq):
        rows = np.nonzero(hit[:, q])[0]
        label = np.full(len(rows), -1, np.int64)
        groups = [np.arange(len(rows))] if rule == 'cross_scene' else \
            [np.nonzero(row_scene[rows] == sc)[0] for sc in np.unique(row_scene[rows])]
        nl = 0
        for gi in groups:
            lab = _components(xyz[rows[gi]], reach, rule)
            label[gi] = lab + nl
            nl += int(lab.max()) + 1 if len(gi) else 0
        size = np.bincount(label, minlength=nl)
        kq = key[rows, q]
        best = np.full(nl, -2, np.int64)
        np.maximum.at(best, label, kq)
        order = np.lexsort((-kq, label))                      # per label, the best hit first
        first = order[np.r_[0, np.nonzero(np.diff(label[order]))[0] + 1]] if len(rows) else order
        brow = np.zeros(nl, np.int64)
        brow[label[first]] = rows[first]
        lo = np.full((nl, 3), np.iinfo(np.int64).max)
        hi = np.full((nl, 3), np.iinfo(np.int64).min)
        np.minimum.at(lo, label, xyz[rows])
        np.maximum.at(hi, label, xyz[rows])
        ok = np.nonzero(size >= min_voxels)[0]
        np.add.at(out['n_regions'][:, q], row_scene[brow[ok]], 1)
        ok = ok[np.lexsort((-best[ok], -size[ok]))] if rule == 'by_size' else ok[np.argsort(-best[ok], kind='stable')]
        rank = np.full(nl + 1, -1, np.int64)
        for j, li in enumerate(ok[:R]):
            b = brow[li]
            rank[li] = j
            out['score'][q, j] = bits[b, q]
            out['scene'][q, j] = row_scene[b]
            out['row'][q, j] = b - off[row_scene[b]]
            out['size'][q, j] = size[li]
            out['box_min'][q, j] = lo[li]
            out['box_max'][q, j] = hi[li]
        hq.append(np.full(len(rows), q, np.int64))
        hr.append(rows)
        hreg.append(rank[label])
    out['score'] = out['score'].view(np.float16)
    hr = np.concatenate(hr) if hr else np.zeros(0, np.int64)
    out['hit_query'] = np.concatenate(hq) if hq else np.zeros(0, np.int64)
    out['hit_scene'] = row_scene[hr]
    out['hit_row'] = hr - off[row_scene[hr]]
    out['hit_score'] = s[hr, out['hit_query']]
    out['hit_region'] = np.concatenate(hreg) if hreg else np.zeros(0, np.int64)
    return out
