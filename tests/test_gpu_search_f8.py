"""The FP8 scene index on the device (DESIGN.md, "FP8 index contract"): the quantizer against tests/f8_ref.py bit for bit,
and every output of ``query`` and ``regions`` on an FP8 index against an fp16 index holding its dequantized rows d, and
against tests/search_ref.py / tests/regions_ref.py on the bits osb_match_scores writes for d."""
import numpy as np
import pytest
import torch

from tests.f8_ref import f8_ref
from tests.regions_ref import regions_ref
from tests.search_ref import search_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _rows(n, c, seed, scale=0.05):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(n, c, generator=g, device=DEV) * scale).half()


def _scores(rows, q):
    from openscene_b200 import matching
    return torch.cat([matching._scores(rows, None, q[i:i + 96].contiguous(), normalize=False)[0]
                      for i in range(0, q.shape[0], 96)], 1)


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


def _offsets(n, layout, rng):
    if layout == 'one':
        return [0, n]
    if layout == 'ones':
        return list(range(n + 1))
    if layout == 'edges':     # boundaries on and around tile edges
        cuts = sorted({x for t in range(128, n, 128) for x in (t - 1, t, t + 1) if 0 < x < n})
        return [0] + cuts + [n]
    if layout == 'tiny':      # thousands of tiny scenes
        cuts = np.sort(rng.choice(np.arange(1, n), min(n - 1, 3000), replace=False))
        return [0] + cuts.tolist() + [n]
    cuts = np.sort(rng.choice(np.arange(1, n), min(n - 1, 7), replace=False))
    return [0] + cuts.tolist() + [n]


def _plant(rows):
    """NaN, inf, zero, saturated (amax above 448 * 2^7), fp16-subnormal and duplicate rows"""
    n = rows.shape[0]
    for i, fill in ((5, float('nan')), (6, 0.0), (n // 2, 0.0)):
        rows[i] = fill
    rows[7, 3] = float('inf')
    rows[8, 5] = float('-inf')
    rows[9, 1] = float('nan')
    rows[10] = (rows[10].float() / rows[10].float().abs().max() * 60000).half()     # amax 60000: e = 7, saturated codes
    rows[11] *= 1e-4                       # fp16 subnormals, e = -15
    rows[12] = rows[n - 3]
    rows[13, :] = 1.0
    rows[13, ::2] = -0.0


def _h(t):
    return None if t is None else (t.view(torch.int16) if t.dtype == torch.float16 else t)


def _same(a, b):
    assert type(a) is type(b)
    for name, x, y in zip(a._fields, a, b):
        assert (x is None) == (y is None), name
        if x is not None:
            assert torch.equal(_h(x), _h(y)), name


def _pair(rows, off, xyz=None, channels=None):
    """an FP8 index of rows and an fp16 index of its dequantized rows d"""
    from openscene_b200.search import SceneIndex
    c = channels or rows.shape[1]
    n = off[-1]
    f8 = SceneIndex(n, c, device=DEV, coords=xyz is not None, storage='fp8')
    f16 = SceneIndex(n, c, device=DEV, coords=xyz is not None)
    xyz_d = None if xyz is None else torch.from_numpy(xyz).to(DEV)
    for a, b in zip(off[:-1], off[1:]):
        f8.add(rows[a:b], coords=None if xyz is None else xyz_d[a:b])
    for s, (a, b) in enumerate(zip(off[:-1], off[1:])):
        f16.add(f8.scene_rows(s), coords=None if xyz is None else xyz_d[a:b])
    d = f16.rows[:n]
    return f8, f16, d


def _check_query(f8, f16, d, off, q, k, thr):
    res = f8.query(q, k=k, threshold=thr)
    _same(res, f16.query(q, k=k, threshold=thr))
    s = _scores(d, q).cpu().numpy()
    ref = search_ref(s, off, k, threshold=None if thr is None else np.full(q.shape[0], thr, np.float32))
    for name in ('score', 'scene', 'row', 'scene_max', 'scene_argmax', 'scene_count'):
        want, got = ref[name], getattr(res, name)
        if want is None:
            assert got is None
            continue
        got = got.cpu().numpy()
        if want.dtype == np.float16:
            want, got = want.view(np.uint16), got.view(np.uint16)
        assert np.array_equal(got, want), name
    return res


def _check_regions(f8, f16, d, xyz, off, q, thr, R=8, reach=1, min_voxels=1):
    res = f8.regions(q, thr, max_regions=R, reach=reach, min_voxels=min_voxels, hits=True)
    _same(res, f16.regions(q, thr, max_regions=R, reach=reach, min_voxels=min_voxels, hits=True))
    s = _scores(d, q).cpu().numpy()
    ref = regions_ref(s, xyz, off, np.full(q.shape[0], thr, np.float32), R, reach, min_voxels)
    for k in ('score', 'scene', 'row', 'size', 'box_min', 'box_max', 'n_regions', 'hit_query', 'hit_scene', 'hit_row',
              'hit_score', 'hit_region'):
        got = getattr(res, k).cpu()
        got = got.view(torch.int16).numpy() if got.dtype == torch.float16 else got.numpy()
        want = ref[k].view(np.int16) if ref[k].dtype == np.float16 else ref[k]
        assert np.array_equal(got, want), k
    return res


# ------------------------------------------------------------------ quantizer

def _quantize(rows):
    from openscene_b200 import _cabi as C
    n, c = rows.shape
    codes = torch.full((n, c), 0xAB, dtype=torch.uint8, device=DEV)
    exps = torch.full((n,), 99, dtype=torch.int8, device=DEV)
    C.call('osb_index_quantize_f8', C.ptr(rows), int(rows.dtype == torch.float16), n, c, C.ptr(codes), C.ptr(exps),
           C.stream_ptr())
    return codes, exps


def _planted_rows(c):
    from tests.test_f8_ref_cpu import _planted
    p = _planted(16)
    out = torch.zeros(p.shape[0], c, dtype=torch.float64)
    out[:, :16] = p
    out[:, c - 16:] = p                                     # the same values in the last lanes' units
    return out


@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32])
@pytest.mark.parametrize('n', [1, 129, 100_003])
def test_quantizer_matches_the_reference(c, dtype, n):
    g = torch.Generator(device=DEV).manual_seed(n + c)
    x = torch.randn(n, c, generator=g, device=DEV, dtype=torch.float32)
    x *= torch.exp(torch.randn(n, 1, generator=g, device=DEV) * 4)          # row scales over many binades
    p = _planted_rows(c).to(DEV, torch.float32)
    m = min(n, p.shape[0])
    x[:m] = p[:m]
    if dtype == torch.float32 and n > 3:
        x[2, 7] = 7e4                                                       # inf as fp16: a NaN row
        x[3, :4] = torch.tensor([1 + 2 ** -12, 1 + 2 ** -11, 1 + 3 * 2 ** -11, 2 ** -25], device=DEV)
    rows = x.to(dtype)
    codes, exps = _quantize(rows)
    rc, re_, _ = f8_ref(rows)
    assert torch.equal(codes, rc)
    assert torch.equal(exps, re_)


def test_quantizer_on_millions_of_rows():
    n, c = 3_000_017, 768
    rows = _rows(n, c, 11, scale=1.0)
    rows[::7] *= 1e-3
    rows[::11] *= 300.0
    codes, exps = _quantize(rows)
    for a in range(0, n, 1 << 20):
        rc, re_, _ = f8_ref(rows[a:a + (1 << 20)])
        assert torch.equal(codes[a:a + (1 << 20)], rc)
        assert torch.equal(exps[a:a + (1 << 20)], re_)


def test_index_rows_are_the_reference_quantization():
    from openscene_b200.search import SceneIndex
    n, c = 20_011, 512
    x = torch.randn(n, c, device=DEV) * 0.05
    idx = SceneIndex(n, c, device=DEV, storage='fp8')
    idx.add(x[:9000])                                  # fp32: .half() first
    idx.add(x[9000:].half())
    rc, re_, rd = f8_ref(x)
    assert torch.equal(idx.codes, rc) and torch.equal(idx.row_exp, re_)
    d = torch.cat([idx.scene_rows(0), idx.scene_rows(1)])
    assert torch.equal(d.view(torch.int16), rd.view(torch.int16))
    assert d.data_ptr() != idx.codes.data_ptr() and idx.rows is None


# ------------------------------------------------------------------ query: FP8 index == fp16 index of d

@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('nq', [1, 20, 96, 200])
def test_query_equals_the_fp16_index_of_d(c, nq):
    n = 30_011
    rows = _rows(n, c, nq)
    _plant(rows)
    off = _offsets(n, 'few', np.random.default_rng(nq))
    f8, f16, d = _pair(rows, off)
    q = _rows(nq, c, 1000 + nq, scale=1.0)
    for k in (1, 2, 7, 32):
        for thr in (None, 0.0, 0.5):
            _check_query(f8, f16, d, off, q, k, thr)


@pytest.mark.parametrize('layout', ['one', 'ones', 'edges', 'tiny'])
def test_query_layouts(layout):
    n = 30_011 if layout != 'ones' else 2000
    rows = _rows(n, 768, 3)
    _plant(rows)
    off = _offsets(n, layout, np.random.default_rng(3))
    f8, f16, d = _pair(rows, off)
    q = _rows(20, 768, 4, scale=1.0)
    _check_query(f8, f16, d, off, q, 8, 0.0)
    _check_query(f8, f16, d, off, q[:1], 32, None)


def test_query_three_million_rows():
    n = 3_000_017
    rows = _rows(n, 768, 5)
    _plant(rows)
    off = _offsets(n, 'few', np.random.default_rng(5))
    f8, f16, d = _pair(rows, off)
    del rows
    _check_query(f8, f16, d, off, _rows(2, 768, 6, scale=1.0), 32, 0.1)
    q = _rows(96, 768, 7, scale=1.0)
    _same(f8.query(q, k=32, threshold=0.1), f16.query(q, k=32, threshold=0.1))


def test_fewer_than_k_scored_rows():
    rows = _rows(40, 768, 1)
    rows[3:] = float('nan')
    rows[1, 5] = float('inf')               # an inf element: the whole FP8 row is NaN
    off = [0, 10, 40]
    f8, f16, d = _pair(rows, off)
    res = _check_query(f8, f16, d, off, _rows(3, 768, 2, scale=1.0), 32, 0.0)
    assert (res.row[:, 2:] == -1).all() and (res.row[:, :2] >= 0).all()


# ------------------------------------------------------------------ regions

@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('nq', [1, 20, 96, 200])
def test_regions_sizes(c, nq):
    n = 20_011
    rows = _rows(n, c, nq)
    _plant(rows)
    off = _offsets(n, 'few', np.random.default_rng(nq))
    xyz = _coords(off, nq)
    f8, f16, d = _pair(rows, off, xyz)
    _check_regions(f8, f16, d, xyz, off, _rows(nq, c, 1000 + nq, scale=1.0), 0.12)


@pytest.mark.parametrize('R', [1, 8, 32])
@pytest.mark.parametrize('reach', [1, 2])
@pytest.mark.parametrize('min_voxels', [1, 3])
def test_regions_parameters(R, reach, min_voxels):
    n = 12_007
    rows = _rows(n, 768, R + reach)
    off = _offsets(n, 'few', np.random.default_rng(R))
    xyz = _coords(off, R + reach, extent=24)
    f8, f16, d = _pair(rows, off, xyz)
    _check_regions(f8, f16, d, xyz, off, _rows(7, 768, 50 + R, scale=1.0), 0.08, R, reach, min_voxels)


@pytest.mark.parametrize('layout', ['one', 'ones', 'edges', 'tiny'])
def test_regions_layouts(layout):
    n = 9001 if layout != 'ones' else 1500
    rows = _rows(n, 512, 0)
    _plant(rows)
    off = _offsets(n, layout, np.random.default_rng(3))
    xyz = _coords(off, 0)
    f8, f16, d = _pair(rows, off, xyz)
    _check_regions(f8, f16, d, xyz, off, _rows(5, 512, 1000, scale=1.0), 0.05, R=16)


# ------------------------------------------------------------------ determinism, streams, memory, host syncs

def test_sentinel_buffers_and_side_stream():
    from openscene_b200 import _cabi as C
    n, c, nq, k = 40_009, 768, 33, 9
    off = [0] + list(range(5000, n, 5000)) + [n]
    rows = _rows(n, c, 8)
    xyz = _coords(off, 8)
    f8, f16, d = _pair(rows, off, xyz)
    q = _rows(nq, c, 9, scale=1.0)
    res = f8.query(q, k=k, threshold=0.08)
    S = f8.n_scenes
    outs = [torch.full((nq, k), 7, dtype=torch.float16, device=DEV)] + \
           [torch.full((nq, k), 7, dtype=torch.int64, device=DEV) for _ in range(2)] + \
           [torch.full((S, nq), 7, dtype=torch.float16, device=DEV)] + \
           [torch.full((S, nq), 7, dtype=torch.int64, device=DEV) for _ in range(2)]
    ws_bytes = C.lib().osb_search_workspace_bytes(S, nq, k)
    ws = torch.full((ws_bytes,), 0xAB, dtype=torch.uint8, device=DEV)
    thr = torch.full((nq,), 0.08, device=DEV)
    off_h = (C.I64 * (S + 1))(*f8._off)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        C.call('osb_search_f8', C.ptr(f8.codes), C.ptr(f8.row_exp), C.ptr(f8.row_scene), n, c, off_h, C.ptr(f8._off_dev),
               S, C.ptr(q), nq, k, C.ptr(thr), *[C.ptr(t) for t in outs], C.ptr(ws), ws_bytes, C.stream_ptr())
        reg_side = f8.regions(q, 0.08, max_regions=9, hits=True)
    torch.cuda.current_stream().wait_stream(side)
    for a, b in zip(res, outs):
        assert torch.equal(_h(a), _h(b))
    _same(res, f8.query(q, k=k, threshold=0.08))
    reg = f8.regions(q, 0.08, max_regions=9, hits=True)
    _same(reg, reg_side)
    _same(reg, f16.regions(q, 0.08, max_regions=9, hits=True))
    # the hit list of osb_search_hits_f8 into sentinel buffers equals the fp16 entry point's on d
    H = len(reg.hit_row)
    lists = []
    for name, operand in (('osb_search_hits_f8', [C.ptr(f8.codes), C.ptr(f8.row_exp)]), ('osb_search_hits', [C.ptr(d)])):
        key = torch.full((H,), 7, dtype=torch.int64, device=DEV)
        hsc = torch.full((H,), 7, dtype=torch.float16, device=DEV)
        st = torch.zeros(1, dtype=torch.int32, device=DEV)
        wsb = C.lib().osb_search_hits_workspace_bytes(S, nq, H)
        ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)
        C.call(name, *operand, C.ptr(f8.row_scene), n, c, off_h, S, C.ptr(q), nq, C.ptr(thr), C.ptr(res.scene_count), H,
               C.ptr(key), C.ptr(hsc), C.ptr(st), C.ptr(ws), wsb, C.stream_ptr())
        assert int(st.item()) == 0
        lists.append((key, hsc.view(torch.int16)))
    assert torch.equal(lists[0][0], lists[1][0]) and torch.equal(lists[0][1], lists[1][1])
    assert torch.equal(lists[0][1], reg.hit_score.view(torch.int16))


def test_add_and_query_make_no_host_synchronisation():
    from openscene_b200.search import SceneIndex
    idx = SceneIndex(20_000, 512, device=DEV, storage='fp8')
    a, b = _rows(5000, 512, 1), torch.randn(3000, 512, device=DEV)
    q = _rows(4, 512, 2, scale=1.0)
    idx.add(a)
    idx.query(q, k=4, threshold=0.0)            # warm the allocator and the module
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        idx.add(a)
        idx.add(b)
        idx.query(q, k=4, threshold=0.0)
        idx.query(q, k=3)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert idx.n_rows == 13_000


@pytest.mark.parametrize('coords', [False, True])
def test_arena_bytes(coords):
    from openscene_b200.search import SceneIndex
    cap, c = 1 << 20, 768
    want = cap * (c + 5) + (16 * cap if coords else 0) + 64 * 8               # + the 64-entry device offsets
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    before = torch.cuda.memory_allocated()
    idx = SceneIndex(cap, c, device=DEV, coords=coords, storage='fp8')
    held = [t for t in vars(idx).values() if isinstance(t, torch.Tensor)]
    assert all(t.is_cuda for t in held) and idx.rows is None
    assert sum(t.untyped_storage().nbytes() for t in held) == want
    # the caching allocator may hand out a cached block up to 1 MiB larger than asked for (it does not split off a
    # remainder of 1 MiB or less), so its count is bounded, not exact
    got = torch.cuda.memory_allocated() - before
    assert want <= got <= want + len(held) * (1 << 20), (got, want)
    del idx, held


def test_peak_memory_under_the_workspace_formula():
    from openscene_b200.search import SceneIndex, search_workspace_bytes
    n, c, nq, k = 5_000_000, 768, 96, 32
    idx = SceneIndex(n, c, device=DEV, storage='fp8')
    per = n // 25
    for s in range(25):
        idx.add(_rows(per, c, s))
    q = _rows(nq, c, 99, scale=1.0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    res = idx.query(q, k=k, threshold=0.1)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    S = idx.n_scenes
    outputs = nq * k * (2 + 8 + 8) + S * nq * (2 + 8 + 8) + 4 * nq + 16 * 512
    assert peak <= search_workspace_bytes(S, nq, k) + outputs + 2 * nq * c + (1 << 20), peak
    assert res.scene_count.sum() > 0


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
    n = sum(len(o) for o in outs)
    f8 = SceneIndex(n, 768, device=DEV, coords=True, storage='fp8')
    f16 = SceneIndex(n, 768, device=DEV, coords=True)
    for o, cc in zip(outs, coords):
        f8.add(o, coords=cc)                          # fp32 rows, MinkowskiEngine (batch, x, y, z) coordinates
    rc, re_, rd = f8_ref(torch.cat(outs))
    assert torch.equal(f8.codes, rc) and torch.equal(f8.row_exp, re_)
    for s, cc in enumerate(coords):
        f16.add(f8.scene_rows(s), coords=cc[:, 1:])
    assert torch.equal(f16.rows.view(torch.int16), rd.view(torch.int16))
    xyz = torch.cat([cc[:, 1:] for cc in coords]).cpu().numpy().astype(np.int32)
    _check_regions(f8, f16, rd, xyz, f8._off, text, 0.0, R=8)
    _check_query(f8, f16, rd, f8._off, text, 4, 0.0)
