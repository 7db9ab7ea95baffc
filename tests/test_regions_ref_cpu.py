"""The region restatement (tests/regions_ref.py) against independent statements of the same contract: a brute-force
breadth-first search, scipy.ndimage.label on dense grids, planted orders and the negative controls."""
from collections import deque

import numpy as np
import pytest
from scipy import ndimage

from tests.regions_ref import regions_ref
from tests.search_ref import order_keys


def _bfs_labels(xyz, reach):
    n = len(xyz)
    lab = np.full(n, -1)
    c = 0
    for s in range(n):
        if lab[s] >= 0:
            continue
        lab[s] = c
        dq = deque([s])
        while dq:
            a = dq.popleft()
            for b in range(n):
                if lab[b] < 0 and np.abs(xyz[a] - xyz[b]).max() <= reach:
                    lab[b] = c
                    dq.append(b)
        c += 1
    return lab


def _cloud(n, extent, seed):
    rng = np.random.default_rng(seed)
    cells = rng.choice(extent ** 3, n, replace=False)
    return np.stack(np.unravel_index(cells, (extent,) * 3), 1).astype(np.int64) - extent // 2


def _same_partition(a, b):
    pa = {}
    for x, y in zip(a, b):
        if pa.setdefault(x, y) != y:
            return False
    return len(set(a)) == len(set(b))


@pytest.mark.parametrize('reach', [1, 2])
@pytest.mark.parametrize('seed', range(4))
def test_against_breadth_first_search(reach, seed):
    xyz = _cloud(150, 12, seed)
    s = np.random.default_rng(seed).standard_normal((150, 1)).astype(np.float16)
    ref = regions_ref(s, xyz, [0, 150], [-np.inf], R=32, reach=reach)
    lab = _bfs_labels(xyz, reach)
    if len(set(lab)) <= 32:
        assert _same_partition(ref['hit_region'], lab)
    sizes = np.bincount(lab)
    assert int(ref['n_regions'].sum()) == len(sizes)
    got = sorted(ref['size'][0][ref['size'][0] > 0].tolist(), reverse=True)
    # the listed sizes are sizes of BFS components; with <= 32 components all are listed
    if len(sizes) <= 32:
        assert got == sorted(sizes.tolist(), reverse=True)
    keys = order_keys(s)[:, 0]
    for j in range(min(32, len(sizes))):
        b = ref['row'][0, j]
        mem = np.nonzero(lab == lab[b])[0]
        assert keys[mem].max() == keys[b]
        assert ref['size'][0, j] == len(mem)
        assert (ref['box_min'][0, j] == xyz[mem].min(0)).all() and (ref['box_max'][0, j] == xyz[mem].max(0)).all()


@pytest.mark.parametrize('seed', range(3))
def test_against_ndimage_label(seed):
    rng = np.random.default_rng(seed)
    grid = rng.random((14, 14, 14)) < 0.2
    lab, n = ndimage.label(grid, structure=np.ones((3, 3, 3)))
    xyz = np.argwhere(grid)
    s = rng.standard_normal((len(xyz), 1)).astype(np.float16)
    ref = regions_ref(s, xyz, [0, len(xyz)], [-np.inf], R=32, reach=1)
    assert ref['n_regions'][0, 0] == n
    dev_lab = lab[tuple(xyz.T)]
    assert _same_partition(ref['hit_region'][ref['hit_region'] >= 0], dev_lab[ref['hit_region'] >= 0])
    listed = ref['size'][0][ref['size'][0] > 0]
    assert set(listed.tolist()) <= set(np.bincount(dev_lab)[1:].tolist())


def test_ties_signed_zero_inf_nan_threshold_and_padding():
    xyz = np.array([[0, 0, 0], [5, 5, 5], [10, 10, 10], [20, 0, 0], [30, 0, 0], [40, 0, 0]])
    s = np.array([[0.5], [0.5], [-0.0], [np.inf], [np.nan], [0.0]], np.float16)
    ref = regions_ref(s, xyz, [0, 3, 6], [0.0], R=8)
    # NaN is never a hit; inf first; the tie 0.5 / 0.5 to the lower row; -0 == +0, the lower global row first
    assert ref['scene'][0].tolist() == [1, 0, 0, 0, 1, -1, -1, -1]
    assert ref['row'][0].tolist() == [0, 0, 1, 2, 2, -1, -1, -1]
    assert ref['score'][0].view(np.uint16)[5:].tolist() == [0xfc00] * 3
    assert ref['size'][0, 5:].tolist() == [0] * 3 and not ref['box_min'][0, 5:].any()
    assert ref['n_regions'][:, 0].tolist() == [3, 2]
    assert 4 not in ref['hit_row'][ref['hit_scene'] == 1]
    none = regions_ref(s, xyz, [0, 3, 6], [np.nan], R=2)
    assert len(none['hit_row']) == 0 and (none['scene'] == -1).all()


def test_min_voxels():
    xyz = np.array([[0, 0, 0], [0, 0, 1], [0, 0, 2], [9, 9, 9]])
    s = np.array([[0.1], [0.2], [0.3], [0.9]], np.float16)
    a = regions_ref(s, xyz, [0, 4], [0.0], R=4, min_voxels=1)
    b = regions_ref(s, xyz, [0, 4], [0.0], R=4, min_voxels=2)
    assert a['size'][0].tolist() == [1, 3, 0, 0] and b['size'][0].tolist() == [3, 0, 0, 0]
    assert b['hit_region'].tolist() == [0, 0, 0, -1] and b['n_regions'][0, 0] == 1


def _planted(seed):
    rng = np.random.default_rng(seed)
    n = 400
    xyz = _cloud(n, 9, seed)
    s = rng.standard_normal((n, 3)).astype(np.float16)
    s[::37] = np.nan
    s[5, 0] = s[300, 0] = 1.0           # a tie across scenes
    xyz[200] = xyz[199] + [0, 1, 1]     # a diagonal neighbour across the scene boundary
    return s, xyz, [0, 200, n]


@pytest.mark.parametrize('rule', ['six', 'by_size', 'tie_high', 'nan_hit', 'cross_scene'])
def test_negative_controls_differ(rule):
    s, xyz, off = _planted(1)
    good = regions_ref(s, xyz, off, [0.2, 0.0, -0.3], R=32, reach=1)
    bad = regions_ref(s, xyz, off, [0.2, 0.0, -0.3], R=32, reach=1, rule=rule)
    assert any(not np.array_equal(good[k].view(np.uint16) if good[k].dtype == np.float16 else good[k],
                                  bad[k].view(np.uint16) if bad[k].dtype == np.float16 else bad[k])
               for k in ('score', 'scene', 'row', 'size', 'n_regions', 'hit_region') if good[k].shape == bad[k].shape) \
        or any(good[k].shape != bad[k].shape for k in good)
