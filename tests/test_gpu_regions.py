"""Regions of search hits on the device (csrc/search.cu hit emission, csrc/regions.cu) against tests/regions_ref.py on the
bits osb_match_scores writes for the same rows and query matrix (slices of at most 96 columns)."""
import numpy as np
import pytest
import torch

from tests.regions_ref import regions_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _scores(rows, q):
    from openscene_b200 import matching
    return torch.cat([matching._scores(rows, None, q[i:i + 96].contiguous(), normalize=False)[0]
                      for i in range(0, q.shape[0], 96)], 1)


def _rows(n, c, seed, scale=0.05):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(n, c, generator=g, device=DEV) * scale).half()


def _coords(off, seed, extent=40):
    """distinct voxels inside every scene"""
    rng = np.random.default_rng(seed)
    out = []
    for a, b in zip(off[:-1], off[1:]):
        n = b - a
        e = max(extent, int(np.ceil((4 * n) ** (1 / 3))))
        cells = rng.choice(e ** 3, n, replace=False)
        out.append(np.stack(np.unravel_index(cells, (e,) * 3), 1) - e // 2)
    return np.concatenate(out).astype(np.int32)


def _index(rows, xyz, off, coords=True):
    from openscene_b200.search import SceneIndex
    idx = SceneIndex(rows.shape[0], rows.shape[1], device=DEV, coords=coords)
    xyz_d = torch.from_numpy(xyz).to(DEV)
    for a, b in zip(off[:-1], off[1:]):
        idx.add(rows[a:b], coords=xyz_d[a:b] if coords else None)
    return idx


def _h(t):
    t = t.cpu()
    return t.view(torch.int16).numpy() if t.dtype == torch.float16 else t.numpy()


def _check(res, ref, hits=True):
    for k in ('score', 'scene', 'row', 'size', 'box_min', 'box_max', 'n_regions'):
        want = ref[k].view(np.int16) if ref[k].dtype == np.float16 else ref[k]
        assert np.array_equal(_h(getattr(res, k)), want), k
    if hits:
        for k in ('hit_query', 'hit_scene', 'hit_row', 'hit_score', 'hit_region'):
            want = ref[k].view(np.int16) if ref[k].dtype == np.float16 else ref[k]
            assert np.array_equal(_h(getattr(res, k)), want), k


def _run(n, c, nq, off, R=8, reach=1, min_voxels=1, thr=0.05, seed=0, hits=True, extent=40):
    rows = _rows(n, c, seed)
    q = _rows(nq, c, seed + 1000, scale=1.0)
    xyz = _coords(off, seed, extent)
    idx = _index(rows, xyz, off)
    res = idx.regions(q, thr, max_regions=R, reach=reach, min_voxels=min_voxels, hits=hits)
    s = _scores(rows, q).cpu().numpy()
    ref = regions_ref(s, xyz, off, np.full(nq, thr, np.float32), R, reach, min_voxels)
    _check(res, ref, hits)
    # invariants: hits per (scene, query) = the search's counts, sizes of all regions sum to the hits
    cnt = idx.query(q, k=1, threshold=thr).scene_count.cpu().numpy()
    hq, hs = ref['hit_query'], ref['hit_scene']
    per = np.zeros_like(cnt)
    np.add.at(per, (hs, hq), 1)
    assert np.array_equal(per, cnt)
    if min_voxels == 1 and R == 32:
        listed = res.size.sum(1).cpu().numpy()
        full = res.n_regions.sum(0).cpu().numpy() <= R
        assert np.array_equal(listed[full], np.bincount(hq, minlength=nq)[full])
    return idx, rows, q, res, ref


def _offsets(n, layout, rng):
    if layout == 'one':
        return [0, n]
    if layout == 'ones':
        return list(range(n + 1))
    if layout == 'edges':
        cuts = sorted({x for t in range(128, n, 128) for x in (t - 1, t, t + 1) if 0 < x < n})
        return [0] + cuts + [n]
    if layout == 'tiny':
        cuts = np.sort(rng.choice(np.arange(1, n), min(n - 1, 3000), replace=False))
        return [0] + cuts.tolist() + [n]
    cuts = np.sort(rng.choice(np.arange(1, n), 5, replace=False))
    return [0] + cuts.tolist() + [n]


@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('nq', [1, 20, 96, 200])
def test_sizes(c, nq):
    n = 20011
    _run(n, c, nq, _offsets(n, 'few', np.random.default_rng(nq)), R=8, thr=0.12, seed=nq)


@pytest.mark.parametrize('R', [1, 8, 32])
@pytest.mark.parametrize('reach', [1, 2])
@pytest.mark.parametrize('min_voxels', [1, 3])
def test_parameters(R, reach, min_voxels):
    n = 12007
    _run(n, 768, 7, _offsets(n, 'few', np.random.default_rng(R)), R=R, reach=reach, min_voxels=min_voxels, thr=0.08,
         seed=R + reach, extent=24)


@pytest.mark.parametrize('layout', ['one', 'ones', 'edges', 'tiny'])
def test_scene_layouts(layout):
    n = 9001 if layout != 'ones' else 1500
    _run(n, 512, 5, _offsets(n, layout, np.random.default_rng(3)), R=16, thr=0.05)


def test_planted_objects_are_found_exactly():
    from openscene_b200.search import SceneIndex
    n_sc, per, c = 6, 3000, 768
    rng = np.random.default_rng(7)
    anchors = torch.nn.functional.normalize(torch.randn(3, c, generator=torch.Generator().manual_seed(7)), dim=1)
    idx = SceneIndex(n_sc * per, c, device=DEV, coords=True)
    boxes = []
    for s in range(n_sc):
        g = np.stack(np.meshgrid(*[np.arange(-15, 15)] * 3, indexing='ij'), -1).reshape(-1, 3)
        lo = rng.integers(-14, 6, 3)
        size = rng.integers(2, 6, 3)
        box = np.all((g >= lo) & (g < lo + size), 1)
        g = np.concatenate([g[box], g[~box][rng.permutation(int((~box).sum()))[:per - int(box.sum())]]])
        g = g[rng.permutation(per)]                          # the whole box and random voxels around it, shuffled
        inside = np.all((g >= lo) & (g < lo + size), 1)
        rows = torch.randn(per, c, generator=torch.Generator().manual_seed(100 + s))
        rows = torch.nn.functional.normalize(rows, dim=1) * 0.02
        a = s % 3
        rows[torch.from_numpy(inside)] = anchors[a]
        idx.add(rows.to(DEV).half(), coords=torch.from_numpy(g).to(DEV))
        boxes.append((a, s, inside.sum(), g[inside].min(0), g[inside].max(0)))
    res = idx.regions(anchors.to(DEV), 0.5, max_regions=4)
    for a in range(3):
        mine = sorted([b for b in boxes if b[0] == a], key=lambda b: b[1])
        got = [(int(res.scene[a, j]), int(res.size[a, j]), res.box_min[a, j].tolist(), res.box_max[a, j].tolist())
               for j in range(4) if res.scene[a, j] >= 0]
        assert sorted(got) == [(s, int(m), lo.tolist(), hi.tolist()) for _, s, m, lo, hi in mine]


def test_top_region_holds_the_top_row():
    n = 30011
    off = _offsets(n, 'few', np.random.default_rng(11))
    idx, rows, q, res, ref = _run(n, 768, 20, off, R=4, thr=0.1, seed=11, hits=False)
    top = idx.query(q, k=1)
    for j in range(q.shape[0]):
        if float(top.score[j, 0]) >= 0.1:
            assert int(res.scene[j, 0]) == int(top.scene[j, 0]) and int(res.row[j, 0]) == int(top.row[j, 0])
            assert torch.equal(res.score[j, 0].view(torch.int16), top.score[j, 0].view(torch.int16))


def test_coords_leave_query_unchanged():
    n = 20000
    off = [0, 7000, 13000, n]
    rows = _rows(n, 768, 4)
    xyz = _coords(off, 4)
    a, b = _index(rows, xyz, off, coords=True), _index(rows, xyz, off, coords=False)
    q = _rows(30, 768, 5, scale=1.0)
    for x, y in zip(a.query(q, k=7, threshold=0.0), b.query(q, k=7, threshold=0.0)):
        assert torch.equal(x, y)


def test_determinism_side_stream_and_sentinel_buffers():
    from openscene_b200 import _cabi as C
    n, c, nq, R = 40009, 768, 33, 9
    off = _offsets(n, 'edges', None)[:1] + list(range(5000, n, 5000)) + [n]
    idx, rows, q, res, ref = _run(n, c, nq, off, R=R, thr=0.08)
    res2 = idx.regions(q, 0.08, max_regions=R, hits=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        res3 = idx.regions(q, 0.08, max_regions=R, hits=True)
    torch.cuda.current_stream().wait_stream(side)
    for a, b, d in zip(res, res2, res3):
        assert torch.equal(a, b) and torch.equal(a, d)
    # the entry points write every output element: sentinel-filled buffers end up equal to the result
    S, H = idx.n_scenes, len(ref['hit_row'])
    thr = torch.full((nq,), 0.08, device=DEV)
    cnt = idx.query(q, k=1, threshold=thr).scene_count
    key = torch.full((H,), 7, dtype=torch.int64, device=DEV)
    hsc = torch.full((H,), 7, dtype=torch.float16, device=DEV)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    wsb = C.lib().osb_search_hits_workspace_bytes(S, nq, H)
    ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)
    C.call('osb_search_hits', C.ptr(idx.rows), C.ptr(idx.row_scene), idx.n_rows, c, (C.I64 * (S + 1))(*idx._off), S,
           C.ptr(q), nq, C.ptr(thr), C.ptr(cnt), H, C.ptr(key), C.ptr(hsc), C.ptr(st), C.ptr(ws), wsb, C.stream_ptr())
    outs = [torch.full((nq, R), 7, dtype=torch.float16, device=DEV)] + \
           [torch.full((nq, R), 7, dtype=torch.int64, device=DEV) for _ in range(3)] + \
           [torch.full((nq, R, 3), 7, dtype=torch.int32, device=DEV) for _ in range(2)] + \
           [torch.full((S, nq), 7, dtype=torch.int64, device=DEV)] + \
           [torch.full((H,), 7, dtype=torch.int64, device=DEV) for _ in range(4)]
    wsb = C.lib().osb_regions_workspace_bytes(H)
    ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)
    C.call('osb_regions', C.ptr(key), C.ptr(hsc), H, C.ptr(idx.coords), C.ptr(idx.row_scene), C.ptr(idx._off_dev),
           idx.n_rows, S, nq, R, 1, 1, *[C.ptr(t) for t in outs], C.ptr(st), C.ptr(ws), wsb, C.stream_ptr())
    assert int(st.item()) == 0
    want = list(res[:7]) + [res.hit_query, res.hit_scene, res.hit_row, res.hit_region]
    for a, b in zip(want, outs):
        assert torch.equal(a, b)
    assert torch.equal(hsc.view(torch.int16), res.hit_score.view(torch.int16))


def test_refusals():
    from openscene_b200.search import SceneIndex
    n, c = 5000, 512
    off = [0, 2000, n]
    rows = _rows(n, c, 1)
    xyz = _coords(off, 1)
    idx = _index(rows, xyz, off)
    q = _rows(3, c, 2, scale=1.0)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(RuntimeError, match=r'\d+ hits exceed max_hits=10'):
        idx.regions(q, -1.0, max_hits=10)
    assert torch.cuda.memory_allocated() - before < 1 << 16          # the counts only, no hit buffers
    # duplicate hit coordinates
    dup = xyz.copy()
    dup[10] = dup[11]
    with pytest.raises(RuntimeError, match='share a voxel'):
        _index(rows, dup, off).regions(q, -1.0)
    # a duplicate among rows that are not hits is not inspected
    rows2 = rows.clone()
    rows2[10] = float('nan')
    _index(rows2, dup, off).regions(q[:1], -1.0)
    far = xyz.copy()
    far[100] = [0, (1 << 17) - 256, 0]
    with pytest.raises(RuntimeError, match='outside'):
        _index(rows, far, off).regions(q, -1.0)
    with pytest.raises(RuntimeError, match='without coordinates'):
        _index(rows, xyz, off, coords=False).regions(q, 0.0)
    plain = SceneIndex(100, c, device=DEV)
    with pytest.raises(ValueError, match='without them'):
        plain.add(rows[:10], coords=torch.zeros(10, 3, dtype=torch.int32, device=DEV))
    with_c = SceneIndex(100, c, device=DEV, coords=True)
    with pytest.raises(ValueError):
        with_c.add(rows[:10])
    with pytest.raises(ValueError):
        with_c.add(rows[:10], coords=torch.zeros(10, 2, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError):
        with_c.add(rows[:10], coords=torch.zeros(9, 3, dtype=torch.int32, device=DEV))
    with pytest.raises(TypeError):
        with_c.add(rows[:10], coords=torch.zeros(10, 3, dtype=torch.float32, device=DEV))
    assert with_c.n_scenes == 0
    for kw in (dict(max_regions=0), dict(max_regions=33), dict(reach=3), dict(min_voxels=0)):
        with pytest.raises(ValueError):
            idx.regions(q, 0.0, **kw)


def test_peak_memory_within_the_per_hit_formula():
    from openscene_b200.search import regions_hit_bytes
    n, c, nq = 400_000, 768, 20
    off = list(range(0, n, 50_000)) + [n]
    rows = _rows(n, c, 3)
    idx = _index(rows, _coords(off, 3, extent=60), off)
    q = _rows(nq, c, 4, scale=1.0)
    idx.regions(q, 0.12, hits=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    res = idx.regions(q, 0.12, hits=True)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    H, S = len(res.hit_row), idx.n_scenes
    assert H > 10_000
    small = S * nq * 8 * 4 + nq * 32 * 64 + (1 << 20)      # counts, search workspace, region outputs, status, queries
    from openscene_b200.search import search_workspace_bytes
    assert peak <= regions_hit_bytes(H, S, nq, hits=True) + search_workspace_bytes(S, nq, 1) + small, (peak, H)


def test_index_of_minkunet_outputs_with_their_coordinates():
    from openscene_b200 import synth
    from openscene_b200 import me as ME
    from openscene_b200.search import SceneIndex
    model = synth.build_model('MinkUNet18A', 768, seed=0).to(DEV).eval()
    text = torch.from_numpy(synth.text_embeddings(20)).to(DEV)
    outs, coords = [], []
    with torch.no_grad():
        for seed in range(3):
            cc = torch.from_numpy(synth.scene('tiny', seed=seed)).to(DEV)      # (batch, x, y, z), unique rows
            feats = torch.rand(len(cc), 3, generator=torch.Generator().manual_seed(seed))
            outs.append(model(ME.SparseTensor(feats.to(DEV), cc)))
            coords.append(cc)
    idx = SceneIndex(sum(len(o) for o in outs), 768, device=DEV, coords=True)
    for o, cc in zip(outs, coords):
        idx.add(o, coords=cc[:, 1:])
    thr = 0.0
    res = idx.regions(text, thr, max_regions=8, reach=1, hits=True)
    rows = torch.cat([o.half() for o in outs])
    s = _scores(rows, text.half()).cpu().numpy()
    xyz = torch.cat([cc[:, 1:] for cc in coords]).cpu().numpy()
    ref = regions_ref(s, xyz, idx._off, np.full(20, thr, np.float32), 8, 1, 1)
    _check(res, ref)
