"""Labelled scene index on the device (SceneIndex.label / labels / class_counts / class_regions; csrc/label.cu, the FP8
instantiation of k_match_tc_topk) against osb_match_topk on the arena rows and the restatements of tests/label_ref.py on
the bits osb_match_scores writes."""
import numpy as np
import pytest
import torch

from tests.label_ref import class_counts_ref, class_regions_ref, label_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _rows(n, c, seed, scale=0.05):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(n, c, generator=g, device=DEV) * scale).half()


def _vocab(K, c, seed):
    v = _rows(K, c, seed, scale=1.0)
    if K >= 8:
        v[5] = v[3]                      # two equal columns: every row ties between them
    return v


def _plant(rows):
    """NaN, inf, zero and tied rows at the start, the middle and the end"""
    n = rows.shape[0]
    for r in (0, n // 2, n - 1):
        rows[r] = 0.0
    for r in (1, n // 2 + 1):
        rows[r, 7] = float('nan')
    for r in (2, n // 2 + 2):
        rows[r, 3] = float('inf')
    if n > 10:
        rows[3] = rows[4]
    return rows


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


def _coords(off, seed, extent=24):
    rng = np.random.default_rng(seed)
    out = []
    for a, b in zip(off[:-1], off[1:]):
        n = b - a
        e = max(extent, int(np.ceil((4 * n) ** (1 / 3))))
        cells = rng.choice(e ** 3, n, replace=False)
        out.append(np.stack(np.unravel_index(cells, (e,) * 3), 1) - e // 2)
    return np.concatenate(out).astype(np.int32)


def _index(rows, off, xyz=None, storage='fp16', capacity=None):
    from openscene_b200.search import SceneIndex
    idx = SceneIndex(capacity or rows.shape[0], rows.shape[1], device=DEV, coords=xyz is not None, storage=storage)
    xyz_d = None if xyz is None else torch.from_numpy(xyz).to(DEV)
    for a, b in zip(off[:-1], off[1:]):
        idx.add(rows[a:b], coords=None if xyz is None else xyz_d[a:b])
    return idx


def _topk1(rows, vocab):
    """osb_match_topk(k = 1) on fp16 rows: (label, score)"""
    from openscene_b200 import _cabi as C
    n = rows.shape[0]
    lab = torch.full((n,), -7, dtype=torch.int64, device=DEV)
    sc = torch.full((n,), 7, dtype=torch.float16, device=DEV)
    C.call('osb_match_topk', C.ptr(rows), 1, n, rows.shape[1], None, n, C.ptr(vocab), vocab.shape[0], 0, 1, C.ptr(sc),
           C.ptr(lab), None, C.stream_ptr())
    return lab, sc


def _scores(rows, vocab):
    from openscene_b200 import matching
    return torch.cat([matching._scores(rows, None, vocab[i:i + 480].contiguous(), normalize=False)[0]
                      for i in range(0, vocab.shape[0], 480)], 1)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t


def _h(t):
    t = t.cpu()
    return t.view(torch.int16).numpy() if t.dtype == torch.float16 else t.numpy()


def _all_labels(idx):
    n = idx.n_rows
    return idx.row_label[:n], idx.row_label_score[:n]


# ------------------------------------------------------------------ labels

@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('K', [1, 20, 96, 97, 160, 480, 1000, 20000])
def test_labels_equal_match_topk(c, K):
    n = 30_011 if K < 20000 else 9_001
    rng = np.random.default_rng(K)
    off = _offsets(n, 'edges' if K % 2 else 'few', rng)
    rows = _plant(_rows(n, c, K))
    vocab = _vocab(K, c, K + 1)
    idx = _index(rows, off)
    idx.label(vocab.float() if K == 20 else vocab)            # fp32 is taken as .half()
    lab, sc = _all_labels(idx)
    want_l, want_s = _topk1(rows, vocab)
    assert torch.equal(lab, want_l) and torch.equal(_bits(sc), _bits(want_s))
    if K <= 480:                                              # the restatement on osb_match_scores' bits
        rl, rs = label_ref(_scores(rows, vocab).cpu().numpy())
        assert np.array_equal(lab.cpu().numpy(), rl)
        assert np.array_equal(_h(sc), rs.view(np.int16))
    # per scene views
    for s in (0, idx.n_scenes - 1):
        a, b = off[s], off[s + 1]
        l, v = idx.labels(s)
        assert torch.equal(l, want_l[a:b]) and torch.equal(_bits(v), _bits(want_s[a:b]))
    # FP8: the labels of the fp16 index holding d
    f8 = _index(rows, off, storage='fp8')
    f8.label(vocab)
    d = torch.cat([f8.scene_rows(s) for s in range(f8.n_scenes)])
    dl, ds = _topk1(d, vocab)
    l8, s8 = _all_labels(f8)
    assert torch.equal(l8, dl) and torch.equal(_bits(s8), _bits(ds))


@pytest.mark.parametrize('layout', ['ones', 'tiny', 'edges'])
def test_label_layouts(layout):
    n = 2000 if layout == 'ones' else 40_000
    off = _offsets(n, layout, np.random.default_rng(5))
    rows = _plant(_rows(n, 768, 5))
    vocab = _vocab(160, 768, 6)
    for storage in ('fp16', 'fp8'):
        idx = _index(rows, off, storage=storage)
        idx.label(vocab)
        src = rows if storage == 'fp16' else torch.cat([idx.scene_rows(s) for s in range(idx.n_scenes)])
        wl, ws = _topk1(src, vocab)
        l, s = _all_labels(idx)
        assert torch.equal(l, wl) and torch.equal(_bits(s), _bits(ws)), storage


def test_three_million_rows():
    n, c = 3_000_017, 768
    off = [0, 128, 129, 1_000_000, 1_000_001, 2_999_999, n]
    rows = _plant(_rows(n, c, 11))
    vocab = _vocab(160, c, 12)
    for storage in ('fp16', 'fp8'):
        idx = _index(rows, off, storage=storage)
        idx.label(vocab)
        src = rows if storage == 'fp16' else torch.cat([idx.scene_rows(s) for s in range(idx.n_scenes)])
        wl, ws = _topk1(src, vocab)
        l, s = _all_labels(idx)
        assert torch.equal(l, wl) and torch.equal(_bits(s), _bits(ws)), storage
        del idx, src


def test_add_labels_its_scene_and_relabel_replaces():
    from openscene_b200.search import SceneIndex
    c = 512
    a, b = _rows(5000, c, 1), _rows(3001, c, 2)
    v1, v2 = _vocab(20, c, 3), _vocab(200, c, 4)
    for storage in ('fp16', 'fp8'):
        idx = SceneIndex(20_000, c, device=DEV, storage=storage)
        idx.label(v1)                                   # empty index: only the vocabulary is stored
        assert idx.n_rows == 0 and idx.row_label is not None
        idx.add(a)
        idx.add(b.float())
        src = torch.cat([idx.scene_rows(s) for s in range(2)])
        wl, ws = _topk1(src, v1)
        l, s = _all_labels(idx)
        assert torch.equal(l, wl) and torch.equal(_bits(s), _bits(ws))
        idx.label(v2)
        wl, ws = _topk1(src, v2)
        l, s = _all_labels(idx)
        assert torch.equal(l, wl) and torch.equal(_bits(s), _bits(ws))
        idx.add(a[:77])
        l, s = idx.labels(2)
        wl, ws = _topk1(idx.scene_rows(2), v2)
        assert torch.equal(l, wl) and torch.equal(_bits(s), _bits(ws))
        assert idx.class_counts().sum().item() == idx.n_rows


# ------------------------------------------------------------------ class counts

@pytest.mark.parametrize('layout', ['few', 'ones', 'tiny', 'edges'])
def test_class_counts(layout):
    n = 1500 if layout == 'ones' else 30_000
    off = _offsets(n, layout, np.random.default_rng(7))
    rows = _plant(_rows(n, 768, 7))
    K = 97
    vocab = _vocab(K, 768, 8)
    vocab[K - 1] = vocab[0]                              # a class no row takes: every tie goes to column 0
    idx = _index(rows, off)
    idx.label(vocab)
    lab, sc = (t.cpu().numpy() for t in _all_labels(idx))
    sc = sc.view(np.float16)
    S = idx.n_scenes
    full = idx.class_counts()
    assert full.shape == (S, K)
    scene_of = torch.repeat_interleave(torch.arange(S, device=DEV), torch.tensor(np.diff(off), device=DEV))
    byhand = torch.bincount(scene_of * K + idx.row_label[:n], minlength=S * K).reshape(S, K)
    assert torch.equal(full, byhand)
    assert np.array_equal(full.cpu().numpy(), class_counts_ref(lab, sc, off, np.arange(K)))
    assert int(full[:, K - 1].sum()) == 0
    classes = [K - 1, 3, 5, 0, 40]
    for thr in (None, 0.0, [0.1, -0.2, 0.05, float('-inf'), 0.3]):
        got = idx.class_counts(classes, threshold=thr).cpu().numpy()
        assert np.array_equal(got, class_counts_ref(lab, sc, off, classes, thr)), thr
    # NaN scores count without a threshold and never with one
    nan_rows = np.isnan(sc.astype(np.float32))
    assert nan_rows.any()
    c0 = idx.class_counts([0]).sum().item()
    c0t = idx.class_counts([0], threshold=float('-inf')).sum().item()
    assert c0 - c0t == int(nan_rows[lab == 0].sum())


def test_class_counts_many_classes_and_tensor_classes():
    n, K = 50_000, 20000
    off = _offsets(n, 'few', np.random.default_rng(9))
    rows = _rows(n, 512, 9)
    idx = _index(rows, off)
    idx.label(_vocab(K, 512, 10))
    lab, sc = (t.cpu().numpy() for t in _all_labels(idx))
    full = idx.class_counts()
    assert np.array_equal(full.cpu().numpy(), class_counts_ref(lab, sc.view(np.float16), off, np.arange(K)))
    pick = torch.tensor([19999, 7, 0], dtype=torch.int32)
    assert torch.equal(idx.class_counts(pick), full[:, [19999, 7, 0]])


# ------------------------------------------------------------------ class regions

def _check_regions(res, ref, hits=True):
    for k in ('score', 'scene', 'row', 'size', 'box_min', 'box_max', 'n_regions'):
        want = ref[k].view(np.int16) if ref[k].dtype == np.float16 else ref[k]
        assert np.array_equal(_h(getattr(res, k)), want), k
    if hits:
        for k in ('hit_query', 'hit_scene', 'hit_row', 'hit_score', 'hit_region'):
            want = ref[k].view(np.int16) if ref[k].dtype == np.float16 else ref[k]
            assert np.array_equal(_h(getattr(res, k)), want), k


def _regions_case(n, c, K, off, seed, storage='fp16', extent=24):
    rows = _plant(_rows(n, c, seed))
    xyz = _coords(off, seed, extent)
    idx = _index(rows, off, xyz, storage=storage)
    idx.label(_vocab(K, c, seed + 1))
    lab, sc = (t.cpu().numpy() for t in _all_labels(idx))
    return idx, xyz, lab, sc.view(np.float16)


@pytest.mark.parametrize('R', [1, 8, 32])
@pytest.mark.parametrize('reach', [1, 2])
@pytest.mark.parametrize('min_voxels', [1, 3])
def test_class_regions_parameters(R, reach, min_voxels):
    n = 12_007
    off = _offsets(n, 'few', np.random.default_rng(R))
    idx, xyz, lab, sc = _regions_case(n, 768, 20, off, R + reach)
    classes = [0, 3, 5, 11, 19]
    for thr in (None, [0.0, -0.05, 0.02, float('-inf'), 0.01]):
        res = idx.class_regions(classes, thr, max_regions=R, reach=reach, min_voxels=min_voxels, hits=True)
        _check_regions(res, class_regions_ref(lab, sc, xyz, off, classes, thr, R, reach, min_voxels))


@pytest.mark.parametrize('m', [1, 20, 96, 200])
def test_class_regions_sizes(m):
    n, K = 20_011, 250
    off = _offsets(n, 'few', np.random.default_rng(m))
    idx, xyz, lab, sc = _regions_case(n, 512, K, off, m, extent=16)
    classes = list(np.random.default_rng(m).permutation(K)[:m])
    for thr in (None, 0.01):
        res = idx.class_regions(classes, thr, max_regions=8, hits=True)
        _check_regions(res, class_regions_ref(lab, sc, xyz, off, classes, thr, 8))
        cnt = idx.class_counts(classes, threshold=float('-inf') if thr is None else thr).cpu().numpy()
        per = np.zeros_like(cnt)
        np.add.at(per, (_h(res.hit_scene), _h(res.hit_query)), 1)
        assert np.array_equal(per, cnt)


@pytest.mark.parametrize('layout', ['ones', 'edges', 'tiny'])
def test_class_regions_layouts_fp8(layout):
    n = 1500 if layout == 'ones' else 9001
    off = _offsets(n, layout, np.random.default_rng(3))
    idx, xyz, lab, sc = _regions_case(n, 768, 20, off, 3, storage='fp8')
    classes = list(range(20))
    res = idx.class_regions(classes, None, max_regions=16, hits=True)
    _check_regions(res, class_regions_ref(lab, sc, xyz, off, classes, None, 16))


def test_query_and_regions_unchanged_on_a_labelled_index():
    n = 20_011
    off = _offsets(n, 'few', np.random.default_rng(4))
    rows = _rows(n, 768, 4)
    xyz = _coords(off, 4)
    q = _rows(30, 768, 5, scale=1.0)
    plain = _index(rows, off, xyz)
    labelled = _index(rows, off, xyz)
    labelled.label(_vocab(160, 768, 6))
    for a, b in zip(plain.query(q, k=9, threshold=0.05), labelled.query(q, k=9, threshold=0.05)):
        assert torch.equal(_bits(a), _bits(b))
    for a, b in zip(plain.regions(q, 0.08, hits=True), labelled.regions(q, 0.08, hits=True)):
        assert torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------ determinism, streams, host syncs, memory

def test_sentinel_buffers_and_side_stream():
    from openscene_b200 import _cabi as C
    n, c, K = 40_009, 768, 160
    off = [0] + list(range(5000, n, 5000)) + [n]
    rows = _plant(_rows(n, c, 8))
    xyz = _coords(off, 8)
    vocab = _vocab(K, c, 9)
    idx = _index(rows, off, xyz, storage='fp8')
    idx.label(vocab)
    lab0, sc0 = (t.clone() for t in _all_labels(idx))
    cnt0 = idx.class_counts()
    classes = [3, 0, 5, 77]
    reg0 = idx.class_regions(classes, 0.0, max_regions=9, hits=True)
    idx.row_label.fill_(-5)
    idx.row_label_score.fill_(7)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        idx.label(vocab)
        cnt1 = idx.class_counts()
        reg1 = idx.class_regions(classes, 0.0, max_regions=9, hits=True)
    torch.cuda.current_stream().wait_stream(side)
    lab1, sc1 = _all_labels(idx)
    assert torch.equal(lab0, lab1) and torch.equal(_bits(sc0), _bits(sc1))
    assert torch.equal(cnt0, cnt1)
    for a, b in zip(reg0, reg1):
        assert torch.equal(_bits(a), _bits(b))
    # osb_label_counts / osb_label_hits into sentinel outputs and workspaces
    S, m = idx.n_scenes, len(classes)
    thr = torch.zeros(m, device=DEV)
    cls = (C.I64 * m)(*classes)
    cnt = torch.full((S, m), 7, dtype=torch.int64, device=DEV)
    wsb = C.lib().osb_label_counts_workspace_bytes(K, m)
    ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)
    C.call('osb_label_counts', C.ptr(idx.row_label), C.ptr(idx.row_label_score), C.ptr(idx.row_scene), n, S, K, cls, m,
           C.ptr(thr), C.ptr(cnt), C.ptr(ws), wsb, C.stream_ptr())
    H = int(cnt.sum())
    assert H == len(reg0.hit_row)
    key = torch.full((H,), 7, dtype=torch.int64, device=DEV)
    hsc = torch.full((H,), 7, dtype=torch.float16, device=DEV)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    wsb = C.lib().osb_label_hits_workspace_bytes(K, n, S, m)
    ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)
    C.call('osb_label_hits', C.ptr(idx.row_label), C.ptr(idx.row_label_score), C.ptr(idx.row_scene), n, S, K, cls, m,
           C.ptr(thr), C.ptr(cnt), H, C.ptr(key), C.ptr(hsc), C.ptr(st), C.ptr(ws), wsb, C.stream_ptr())
    assert int(st.item()) == 0
    row0 = torch.tensor(idx._off[:-1], device=DEV)[reg0.hit_scene]
    assert torch.equal(key, (reg0.hit_query << 32) | (row0 + reg0.hit_row))
    assert torch.equal(_bits(hsc), _bits(reg0.hit_score))
    # counts that do not match the labels raise the status bit
    cnt[0, 0] += 1
    st.zero_()
    key = torch.empty(H + 1, dtype=torch.int64, device=DEV)
    hsc = torch.empty(H + 1, dtype=torch.float16, device=DEV)
    C.call('osb_label_hits', C.ptr(idx.row_label), C.ptr(idx.row_label_score), C.ptr(idx.row_scene), n, S, K, cls, m,
           C.ptr(thr), C.ptr(cnt), H + 1, C.ptr(key), C.ptr(hsc), C.ptr(st), C.ptr(ws), wsb, C.stream_ptr())
    assert int(st.item()) & 1


def test_label_add_and_class_counts_make_no_host_synchronisation():
    from openscene_b200.search import SceneIndex
    for storage in ('fp16', 'fp8'):
        idx = SceneIndex(20_000, 512, device=DEV, storage=storage)
        a, b = _rows(5000, 512, 1), torch.randn(3000, 512, device=DEV)
        v = _vocab(160, 512, 2)
        idx.add(a)
        idx.label(v)
        idx.class_counts([3, 1], threshold=0.0)       # warm the allocator and the modules
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            idx.label(v)
            idx.add(a)
            idx.add(b)
            idx.class_counts()
            idx.class_counts([3, 1], threshold=[0.0, 0.1])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert idx.class_counts().sum().item() == 13_000


def test_arena_bytes_and_peak_memory():
    from openscene_b200.search import SceneIndex
    cap, c, K = 1 << 21, 768, 1000
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    idx = SceneIndex(cap, c, device=DEV, coords=True)
    held = sum(t.untyped_storage().nbytes() for t in vars(idx).values() if isinstance(t, torch.Tensor))
    per = cap // 8
    rows = _rows(per, c, 1)
    xyz = torch.from_numpy(_coords([0, per], 1)).to(DEV)
    for _ in range(8):
        idx.add(rows, coords=xyz)
    del rows
    vocab = _vocab(K, c, 2)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    idx.label(vocab)
    torch.cuda.synchronize()
    labelled = sum(t.untyped_storage().nbytes() for t in vars(idx).values() if isinstance(t, torch.Tensor))
    assert labelled == held + 10 * cap + K * c * 2            # 10 B per row and the vocabulary copy
    assert torch.cuda.max_memory_allocated() - base <= 10 * cap + K * c * 2 + (4 << 20)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    cnt = idx.class_counts()
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= 8 * K * 8 + 12 * K + (2 << 20)
    assert int(cnt.sum()) == cap
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    res = idx.class_regions([0, 1, 2], 0.05, hits=False)
    torch.cuda.synchronize()
    H = int(idx.class_counts([0, 1, 2], threshold=0.05).sum())
    from openscene_b200 import _cabi as CA
    ws = max(CA.lib().osb_label_hits_workspace_bytes(K, cap, 8, 3), CA.lib().osb_regions_workspace_bytes(H))
    assert torch.cuda.max_memory_allocated() - base <= 10 * H + ws + (4 << 20)
    assert res.n_regions.sum() > 0


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
    off = np.cumsum([0] + [len(o) for o in outs])
    for storage in ('fp16', 'fp8'):
        idx = SceneIndex(n, 768, device=DEV, coords=True, storage=storage)
        idx.label(text)
        for o, cc in zip(outs, coords):
            idx.add(o, coords=cc)                         # fp32 rows, labelled as they are added
        src = torch.cat([idx.scene_rows(s) for s in range(idx.n_scenes)])
        wl, ws = _topk1(src, text)
        lab, sc = _all_labels(idx)
        assert torch.equal(lab, wl) and torch.equal(_bits(sc), _bits(ws))
        # on NaN-free rows the label is evaluate.py's torch.max(pred, 1)[1] of the fp16 scores
        s = _scores(src, text)
        assert torch.equal(lab, s.float().cpu().max(1)[1].to(DEV))
        xyz = torch.cat([cc[:, 1:] for cc in coords]).cpu().numpy().astype(np.int32)
        l_np, s_np = lab.cpu().numpy(), sc.cpu().numpy().view(np.float16)
        res = idx.class_regions(list(range(20)), None, max_regions=8, hits=True)
        _check_regions(res, class_regions_ref(l_np, s_np, xyz, off, list(range(20)), None, 8))
        assert np.array_equal(idx.class_counts().cpu().numpy(), class_counts_ref(l_np, s_np, off, np.arange(20)))


def test_refusals():
    from openscene_b200.search import SceneIndex
    idx = SceneIndex(1000, 512, device=DEV)
    idx.add(_rows(100, 512, 1))
    with pytest.raises(RuntimeError, match='not labelled'):
        idx.labels(0)
    with pytest.raises(RuntimeError, match='not labelled'):
        idx.class_counts()
    for bad, err in ((_rows(4, 768, 1), ValueError), (_rows(4, 512, 1).bfloat16(), TypeError),
                     (_rows(4, 512, 1).cpu(), ValueError), (_rows(0, 512, 1), ValueError),
                     (_rows(4, 512, 1)[0], ValueError)):
        with pytest.raises(err):
            idx.label(bad)
    assert idx.vocab is None
    idx.label(_vocab(10, 512, 2))
    with pytest.raises(RuntimeError, match='coordinates'):
        idx.class_regions([0])
    with pytest.raises(ValueError, match='thresholds'):
        idx.class_counts([0, 1], threshold=[0.1, 0.2, 0.3])
    with pytest.raises(ValueError, match='listed twice'):
        idx.class_counts([1, 1])
    with pytest.raises(ValueError, match='outside'):
        idx.class_counts([10])
    big = SceneIndex(2000, 512, device=DEV)
    for _ in range(1025):
        big.add(_rows(1, 512, 3))
    big.label(_vocab(1 << 17, 512, 4))
    with pytest.raises(ValueError, match='exceed'):
        big.class_counts()                              # 1,025 scenes x 2^17 classes: above 2^27 counts
    assert big.class_counts(range(1 << 10)).shape == (1025, 1 << 10)
