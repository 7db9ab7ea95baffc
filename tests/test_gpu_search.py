"""Scene search on the device (csrc/search.cu) against tests/search_ref.py on the bits osb_match_scores writes for the
same rows and query matrix (at most 96 columns, so column positions match)."""
import numpy as np
import pytest
import torch

from tests.search_ref import search_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _index(rows, off):
    from openscene_b200.search import SceneIndex
    idx = SceneIndex(rows.shape[0], rows.shape[1], device=DEV)
    for a, b in zip(off[:-1], off[1:]):
        idx.add(rows[a:b])
    return idx


def _scores(rows, q):
    from openscene_b200 import matching
    s, _, _ = matching._scores(rows, None, q, normalize=False)
    return s


def _rows(n, c, seed, scale=0.05):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(n, c, generator=g, device=DEV) * scale).half()


def _check(res, ref, s_gpu):
    h = lambda t: t.cpu().numpy()
    assert np.array_equal(h(res.score).view(np.uint16), ref['score'].view(np.uint16))
    assert np.array_equal(h(res.scene), ref['scene'])
    assert np.array_equal(h(res.row), ref['row'])
    assert np.array_equal(h(res.scene_max).view(np.uint16), ref['scene_max'].view(np.uint16))
    assert np.array_equal(h(res.scene_argmax), ref['scene_argmax'])
    if ref['scene_count'] is not None:
        assert np.array_equal(h(res.scene_count), ref['scene_count'])


def _run(n, c, nq, k, off, seed=0, plant=None, thr=0.0):
    rows = _rows(n, c, seed)
    if plant is not None:
        plant(rows)
    q = _rows(nq, c, seed + 1000, scale=1.0)
    idx = _index(rows, off)
    res = idx.query(q, k=k, threshold=thr)
    s = _scores(rows, q)
    ref = search_ref(s.cpu().numpy(), off, k, threshold=None if thr is None else np.full(nq, thr, np.float32))
    # every returned score is the matrix's bits at its (row, q)
    sc, sr = res.scene.cpu(), res.row.cpu()
    ok = sc >= 0
    grow = torch.tensor(off)[sc.clamp(min=0)] + sr
    qq = torch.arange(nq)[:, None].expand_as(sc)
    got = res.score.cpu().view(torch.int16)[ok]
    assert torch.equal(got, s.cpu().view(torch.int16)[grow[ok], qq[ok]])
    _check(res, ref, s)
    return idx, rows, q, res


def _offsets(n, layout, rng):
    if layout == 'one':
        return [0, n]
    if layout == 'ones':
        return list(range(n + 1))
    if layout == 'edges':     # boundaries on and around tile edges
        cuts = sorted({x for t in range(128, n, 128) for x in (t - 1, t, t + 1) if 0 < x < n})
        return [0] + cuts + [n]
    if layout == 'tiny':      # ~10k tiny scenes
        cuts = np.sort(rng.choice(np.arange(1, n), min(n - 1, 10000), replace=False))
        return [0] + cuts.tolist() + [n]
    cuts = np.sort(rng.choice(np.arange(1, n), min(n - 1, 7), replace=False))
    return [0] + cuts.tolist() + [n]


@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('n', [1, 63, 64, 65, 127, 128, 129, 100003])
@pytest.mark.parametrize('nq,k', [(1, 1), (2, 2), (95, 31), (96, 32)])
def test_sizes(n, c, nq, k):
    rng = np.random.default_rng(n + nq)
    _run(n, c, nq, k, _offsets(n, 'few', rng), seed=n)


@pytest.mark.parametrize('layout', ['one', 'ones', 'edges', 'tiny'])
def test_scene_layouts(layout):
    n = 30011 if layout != 'ones' else 2000
    _run(n, 768, 20, 8, _offsets(n, layout, np.random.default_rng(3)))


def test_three_million_rows():
    n = 3_000_017
    _run(n, 768, 2, 32, _offsets(n, 'few', np.random.default_rng(5)), seed=5)


def test_edge_rows():
    n = 50000

    def plant(rows):
        rows[1000] = rows[40000]             # duplicates in different scenes and tiles
        rows[129] = rows[40000]
        rows[77] = 0
        rows[5] = float('nan')
        rows[6, 3] = float('inf')
        rows[7, 3] = float('-inf')
        rows[300:400] = float('nan')         # a whole scene of NaN

    off = [0, 200, 300, 400, 10000, 30000, n]
    _run(n, 512, 96, 32, off, plant=plant)


def test_fewer_than_k_scored_rows():
    def plant(rows):
        rows[3:] = float('nan')
    _run(40, 768, 3, 32, [0, 10, 40], plant=plant)


def test_outputs_in_sentinel_buffers_and_determinism():
    from openscene_b200 import _cabi as C
    n, c, nq, k = 70001, 768, 33, 9
    off = _offsets(n, 'edges', None)[:1] + list(range(5000, n, 5000)) + [n]
    idx, rows, q, res = _run(n, c, nq, k, off)
    S = idx.n_scenes
    outs = [torch.full((nq, k), 7, dtype=torch.float16, device=DEV), torch.full((nq, k), 7, dtype=torch.int64, device=DEV),
            torch.full((nq, k), 7, dtype=torch.int64, device=DEV), torch.full((S, nq), 7, dtype=torch.float16, device=DEV),
            torch.full((S, nq), 7, dtype=torch.int64, device=DEV), torch.full((S, nq), 7, dtype=torch.int64, device=DEV)]
    ws_bytes = C.lib().osb_search_workspace_bytes(S, nq, k)
    ws = torch.full((ws_bytes,), 0xAB, dtype=torch.uint8, device=DEV)
    thr = torch.zeros(nq, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        C.call('osb_search', C.ptr(idx.rows), C.ptr(idx.row_scene), idx.n_rows, c, (C.I64 * (S + 1))(*idx._off),
               C.ptr(idx._off_dev), S, C.ptr(q), nq, k, C.ptr(thr), *[C.ptr(t) for t in outs], C.ptr(ws), ws_bytes,
               C.stream_ptr())
    torch.cuda.current_stream().wait_stream(side)
    for a, b in zip(res, outs):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a,
                           b.view(torch.int16) if b.dtype == torch.float16 else b)
    res2 = idx.query(q, k=k, threshold=0.0)
    for a, b in zip(res, res2):
        assert torch.equal(a, b)


def test_peak_memory_under_the_workspace_formula():
    from openscene_b200.search import SceneIndex, search_workspace_bytes
    n, c, nq, k = 5_000_000, 768, 96, 32
    idx = SceneIndex(n, c, device=DEV)
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
    assert peak < n * nq * 2 / 100
    assert res.scene_count.sum() > 0


def test_query_makes_no_host_synchronisation():
    rows = _rows(5000, 512, 1)
    idx = _index(rows, [0, 1000, 5000])
    q = _rows(4, 512, 2, scale=1.0)
    idx.query(q, k=4, threshold=0.0)            # warm the allocator and the module
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        idx.query(q, k=4, threshold=0.0)
        idx.query(q, k=3)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_more_than_96_queries_slice():
    n, c = 20000, 768
    rows = _rows(n, c, 4)
    off = [0, 7000, 13000, n]
    idx = _index(rows, off)
    q = _rows(200, c, 5, scale=1.0)
    full = idx.query(q, k=5, threshold=0.0)
    parts = [idx.query(q[a:b], k=5, threshold=0.0) for a, b in ((0, 96), (96, 192), (192, 200))]
    for j in range(3):
        assert torch.equal(full[j], torch.cat([p[j] for p in parts], 0))
    for j in range(3, 6):
        assert torch.equal(full[j], torch.cat([p[j] for p in parts], 1))


def test_index_of_minkunet_outputs_matches_the_matching_path():
    from openscene_b200 import matching, synth
    from openscene_b200 import me as ME
    from openscene_b200.search import SceneIndex
    model = synth.build_model('MinkUNet18A', 768, seed=0).to(DEV).eval()
    text = torch.from_numpy(synth.text_embeddings(20)).to(DEV)
    outs = []
    with torch.no_grad():
        for seed in range(3):
            coords = synth.random_cloud(1500 + 300 * seed, 24, seed=seed)
            feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(seed))
            outs.append(model(ME.SparseTensor(feats.to(DEV), torch.from_numpy(coords).to(DEV))))
    idx = SceneIndex(sum(len(o) for o in outs), 768, device=DEV)
    ens = SceneIndex(sum(len(o) for o in outs), 768, device=DEV)
    fused = [torch.randn(len(o), 768, device=DEV).half() for o in outs]
    for o, f in zip(outs, fused):
        idx.add(o)                                   # fp32: the 'distill' operand, .half()
        _, _, fe, _ = matching.match_ensemble(o, f, None, text, return_features=True)
        ens.add(fe)
    res = idx.query(text, k=4)
    res_e = ens.query(text, k=4)
    for s, (o, f) in enumerate(zip(outs, fused)):
        sc, _ = matching.match_distill(o, None, text)
        assert torch.equal(res.scene_max[s].view(torch.int16), sc.max(0).values.view(torch.int16))
        se, _, _, _ = matching.match_ensemble(o, f, None, text)
        assert torch.equal(res_e.scene_max[s].view(torch.int16), se.max(0).values.view(torch.int16))
