"""osb_match_topk / osb_match_ensemble_topk (k_match_tc_topk) and matching.match_topk / match_ensemble_topk on the GPU.

The expected scores come from osb_match_scores run on 480-row slices of the text matrix: 480 = 5 x 96, so every column
keeps its position within its 96-row pass, and the kernel's scores must be the same bits.  The expected top-k applies
tests/topk_ref.py to them slice by slice and merges the slices' results by the same rule.  Every output lands in a
sentinel-filled buffer.  Also: labels[:, 0] and smax against osb_match_scores (finite rows) and osb_match_ce (rows with a
NaN) for K <= 480, edge rows, the ensemble against match_ensemble and against its chunked restatement, the label sets of
torch's fp16 product where the fp64 gap between the k-th and the (k+1)-th score exceeds the per-score bounds, peak memory
at K = 20,000 on a config2_200k scene, 1,366 passes, and identical bits over two runs and on a side stream."""
import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import matching, synth
from tests import match_ref as M
from tests import topk_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SLICE = 480
KS = [1, 2, 95, 96, 97, 480, 481, 1203, 4096, 20011]
NPTS = [1, 127, 129, 100003]


def _text(k, c, seed=0):
    return torch.from_numpy(synth.text_embeddings(k, c, seed)).to(DEV)


def _feats(n, c, g, f16=False):
    f = (torch.randn(n, c, generator=g) * (0.2 + torch.rand(n, 1, generator=g))).to(DEV)
    return f.half() if f16 else f


def _inds(n_pts, g):
    """a permutation of about half as many voxels with repeats, shuffled: (n_vox, inds_reverse)"""
    n_vox = n_pts // 2 + 1
    inv = torch.cat([torch.randperm(n_vox, generator=g), torch.randint(0, n_vox, (max(0, n_pts - n_vox),), generator=g)])
    return n_vox, inv[torch.randperm(inv.shape[0], generator=g)][:n_pts].to(DEV)


def bits(x):
    return x.view(torch.int16)


def same_bits(a, b):
    """equal fp16 bits, any NaN equal to any NaN"""
    return bool(((bits(a) == bits(b)) | (torch.isnan(a.float()) & torch.isnan(b.float()))).all())


def topk_call(feat, inv, text, k, normalize, stream=None):
    """one osb_match_topk into sentinel-filled buffers: (scores, labels, smax)"""
    n_pts = inv.shape[0] if inv is not None else feat.shape[0]
    scores = torch.full((n_pts, k), -1234.0, dtype=torch.float16, device=DEV)
    label = torch.full((n_pts, k), -7, dtype=torch.int64, device=DEV)
    smax = torch.full((n_pts,), float('nan'), dtype=torch.float32, device=DEV)
    s = C.stream_ptr() if stream is None else C.c_void_p(stream.cuda_stream)
    C.call('osb_match_topk', C.ptr(feat), int(feat.dtype == torch.float16), feat.shape[0], feat.shape[1], C.ptr(inv), n_pts,
           C.ptr(text), text.shape[0], int(normalize), k, C.ptr(scores), C.ptr(label), C.ptr(smax), s)
    return scores, label, smax


def expected(feat, inv, text, k, normalize, got=None):
    """the chunked restatement: (labels, scores, smax) from osb_match_scores on 480-row slices; with got = (scores, labels) of
    the kernel, also checks that each of its scores is the slice run's score at the same column, bit for bit"""
    K = text.shape[0]
    cols, vals, smax = [], [], None
    for j in range(0, K, SLICE):
        s, _, m = matching._scores(feat, inv, text[j:j + SLICE], normalize, want_smax=True)
        w = s.shape[1]
        if got is not None:
            gs, gl = got
            inside = (gl >= j) & (gl < j + w)
            at = s.gather(1, (gl - j).clamp(0, w - 1))
            assert same_bits(at[inside], gs[inside]), f"a score differs from the slice run at its column (slice {j})"
        lab, sc = R.topk_torch(s, min(k, w))
        cols.append(lab + j)
        vals.append(sc)
        smax = m if smax is None else torch.where(m > smax, m, smax)      # equal maxima: the lower slice's
    lab, sc = R.topk_torch(torch.cat(vals, 1), k, torch.cat(cols, 1))
    return lab, sc, smax


def check(feat, inv, text, k, normalize):
    s, l, m = topk_call(feat, inv, text, k, normalize)
    el, es, em = expected(feat, inv, text, k, normalize, got=(s, l))
    assert torch.equal(l, el), f"labels differ at {int((l != el).any(1).nonzero()[0])}"
    assert same_bits(s, es)
    assert torch.equal(m.view(torch.int32), em.view(torch.int32))
    return s, l, m


def cases(K):
    """per K both widths; across the list every n_pts, dtype, normalize and inds_reverse pairing"""
    i = KS.index(K)
    return [(c, NPTS[(i + j) % 4], (i + j) % 2 == 1, (i // 2 + j) % 2 == 1, (i + 2 * j) % 3 != 0)
            for j, c in enumerate((512, 768))]


@pytest.mark.parametrize('K', KS)
def test_scores_and_labels_bit_for_bit(K):
    g = torch.Generator().manual_seed(K)
    for c, n_pts, f16, normalize, use_inv in cases(K):
        n_vox, inv = _inds(n_pts, g) if use_inv else (n_pts, None)
        feat = _feats(n_vox, c, g, f16)
        text = _text(K, c, seed=K % 7)
        for k in sorted({1, 3, 8} & set(range(1, K + 1))):
            s, l, m = check(feat, inv, text, k, normalize)
            if K <= SLICE:      # finite rows: labels[:, 0] and smax are osb_match_scores'
                _, l0, m0 = matching._scores(feat, inv, text, normalize, want_scores=False, want_smax=True)
                assert torch.equal(l[:, 0], l0) and torch.equal(m.view(torch.int32), m0.view(torch.int32))


@pytest.mark.parametrize('K', [97, 480])
def test_rows_with_nan_follow_the_validation_argmax(K):
    """a NaN in text row j makes column j NaN for every point: labels[:, 0] is osb_match_ce's prediction"""
    from tests.test_gpu_match_ce import match_ce
    g = torch.Generator().manual_seed(5)
    feat = _feats(3000, 768, g)
    text = _text(K, 768)
    text[K // 3, 17] = float('nan')
    y = torch.randint(0, K, (3000,), generator=g).to(DEV)
    _, pred, _, _, _ = match_ce(feat, None, text, y, K)
    for k in (1, 4):
        s, l, m = check(feat, None, text, k, False)
        assert torch.equal(l[:, 0], pred) and bool((l[:, 0] == K // 3).all())


def test_edge_rows():
    """duplicate text rows (equal scores: the lower column first), zero feature rows (+-0), huge rows (fp16 +-inf) and a
    NaN row (all NaN: labels 0..k-1)"""
    g = torch.Generator().manual_seed(9)
    K, c = 1203, 768
    text = _text(K, c)
    text[600:700] = text[100:200]                   # twins in another pass and another slice
    text[5] = text[2]
    feat = _feats(512, c, g)
    feat[10:20] = 0.0
    feat[20:30] = -0.0
    sign = torch.sign(text[7].float())
    feat[30:35] = 3e4 * sign                         # fp16-finite operands whose products overflow: +inf at column 7
    feat[35:40] = -3e4 * sign
    feat[40, 3] = float('nan')
    for k in (1, 3, 8):
        for normalize in (False, True):
            s, l, m = check(feat, None, text, k, normalize)
            assert torch.equal(l[40], torch.arange(k, device=DEV)) and bool(torch.isnan(s[40].float()).all())
            assert float(m[40]) == float('-inf')
            assert torch.equal(l[10:30], torch.arange(k, device=DEV).expand(20, k)) and bool((s[10:30] == 0).all())
            if not normalize:
                assert bool(torch.isinf(s[30:40].float()).any())
            lc, sc = l.cpu().tolist(), s.float().cpu().tolist()
            for lr, sr in zip(lc, sc):              # of two equal twins, the lower column ranks first
                for a, b in [(2, 5)] + [(x, x + 500) for x in range(100, 200)]:
                    if a in lr and b in lr and sr[lr.index(a)] == sr[lr.index(b)]:
                        assert lr.index(b) > lr.index(a)


def ensemble_expected(pred, f2, inv, text, k):
    """chunked restatement of match_ensemble_topk: slice maxima combined by the kernel's rule, the choice, then the chunked
    top-k of the chosen operand"""
    _, _, m2 = expected(f2, inv, text, 1, True)
    _, _, m3 = expected(pred, inv, text, 1, True)
    mask = m3 < m2
    rows = inv if inv is not None else torch.arange(pred.shape[0], device=DEV)
    fe = torch.where(mask[:, None], f2[rows], pred[rows].half())
    lab, sc, _ = expected(fe, None, text, k, False)
    return lab, sc, fe, mask


@pytest.mark.parametrize('K', [160, 480, 1203, 20011])
def test_ensemble(K):
    g = torch.Generator().manual_seed(K + 1)
    c = 768 if K % 2 else 512
    n_vox, inv = _inds(4099, g)
    pred = _feats(n_vox, c, g)
    f2 = _feats(n_vox, c, g, f16=True)
    text = _text(K, c)
    for k in (1, 5):
        s, l, fe, mask = matching.match_ensemble_topk(pred, f2, inv, text, k=k, return_features=True)
        assert s.shape == (4099, k) and l.shape == (4099, k) and fe.shape == (4099, c)
        if K <= SLICE:
            s0, l0, fe0, mask0 = matching.match_ensemble(pred, f2, inv, text, return_features=True)
            assert torch.equal(mask, mask0) and torch.equal(bits(fe), bits(fe0)) and torch.equal(l[:, 0], l0)
            assert torch.equal(bits(s), bits(s0.gather(1, l)))
        el, es, efe, emask = ensemble_expected(pred, f2, inv, text, k)
        assert torch.equal(mask, emask) and torch.equal(bits(fe), bits(efe))
        assert torch.equal(l, el) and same_bits(s, es)


def test_agrees_with_the_reference_product():
    """K = 1203: every score within the fp64 per-score bound (tests/match_ref.py); where the fp64 k-th and (k+1)-th scores
    are further apart than their bounds and torch's own error, the label set is torch's ``(X[inv].half() @ T.t()).topk(k)``"""
    g = torch.Generator().manual_seed(11)
    K, c = 1203, 768
    n_vox, inv = _inds(20000, g)
    x = _feats(n_vox, c, g)
    text = _text(K, c)
    coeff = M.acc_coeff('tc', c)
    ref = (x[inv].half() @ text.t())
    for k in (1, 5, 8):
        s, l = matching.match_topk(x, inv, text, k=k)
        a = M.operand(x[inv], False)
        S, A, E = M.reference(a, text)
        B = M.bound(S, A, E, coeff)
        assert M.score_ratio(s, S.gather(1, l), B.gather(1, l)) <= 1.0
        Ss, order = S.sort(dim=1, descending=True)
        Bs = B.gather(1, order)
        sep = (Ss[:, k - 1] - Ss[:, k]) > 2 * (Bs[:, k - 1] + Bs[:, k])
        assert int(sep.sum()) > 0.5 * sep.numel()
        tl = ref.topk(k, dim=1).indices
        assert torch.equal(l[sep].sort(1).values, tl[sep].sort(1).values)


def _scene_points(name):
    pts, voxel = synth.scene_points(name)
    vox = np.floor(pts / voxel).astype(np.int64)
    _, inv = np.unique(vox, axis=0, return_inverse=True)
    return int(inv.max()) + 1, torch.from_numpy(inv.reshape(-1)).to(DEV)


def test_memory_does_not_grow_with_the_vocabulary():
    """config2_200k points at K = 20,000, k = 5: the [N_pts, K] scores (about 18 GB) never exist"""
    n_vox, inv = _scene_points('config2_200k')
    g = torch.Generator().manual_seed(3)
    x = _feats(n_vox, 768, g)
    text = _text(20000, 768)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    s, l = matching.match_topk(x, inv, text, k=5)
    torch.cuda.synchronize()
    out = s.numel() * 2 + l.numel() * 8
    assert torch.cuda.max_memory_allocated() - base <= out + 64 * 2 ** 20
    assert s.shape == (inv.shape[0], 5) and bool(((l >= 0) & (l < 20000)).all())
    rows = torch.randperm(inv.shape[0], generator=g)[:300].to(DEV)
    el, es, _ = expected(x, inv[rows], text, 5, False)
    assert torch.equal(l[rows], el) and same_bits(s[rows], es)


def test_many_passes():
    """K = 131,072 at 1,000 points: 1,366 passes, so the text ring's barrier parity wraps hundreds of times"""
    g = torch.Generator().manual_seed(4)
    text = _text(131072, 512)
    feat = _feats(1000, 512, g, f16=True)
    for k in (1, 8):
        check(feat, None, text, k, k == 8)


def test_two_runs_and_a_side_stream_give_the_same_bits():
    g = torch.Generator().manual_seed(6)
    n_vox, inv = _inds(30000, g)
    feat = _feats(n_vox, 768, g)
    text = _text(2000, 768)
    a = topk_call(feat, inv, text, 8, True)
    b = topk_call(feat, inv, text, 8, True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = topk_call(feat, inv, text, 8, True, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for x, y in ((a, b), (a, c)):
        assert torch.equal(bits(x[0]), bits(y[0])) and torch.equal(x[1], y[1]) and torch.equal(x[2].view(torch.int32),
                                                                                                y[2].view(torch.int32))
