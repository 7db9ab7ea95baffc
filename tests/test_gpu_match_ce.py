"""osb_match_ce (k_match_tc_ce) and DeviceValidation on the GPU: the validation tail of run/distill.py (:419-446).

Per case: the scores are bit-identical to osb_match_scores, pred equals torch CUDA's ``scores.max(1)[1]`` (finite rows,
rows with one NaN), the counts equal intersectionAndUnionGPU (restated in tests/valce_ref.py) exactly, each row's
log-probability at its label is within the bound of valce_ref.logp_bound (the fp32 error before the final rounding) plus
half an fp16 ulp of the fp64 value T (one fp16 ulp of fp16(T) where that fp32 error is below half an ulp), torch CUDA's
log_softmax within the same bound, and the scene loss within valce_ref.loss_bound of the fp64 mean and of torch's
``F.cross_entropy(scores, label, ignore_index=255)``.  Every output lands in a NaN- (or sentinel-) filled buffer; two runs
give the same bits.  A row's log-probability is read through the loss of a scene in which only that row is labelled.

End to end: FusedMinkUNet(model, batch_stats=True) outputs of config1_50k scenes fed to the restated torch tail (with its
.cpu() reads) and to DeviceValidation give identical mIoU / mAcc / allAcc and loss_avg within the loss bound."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from openscene_b200 import _cabi as C
from openscene_b200 import distill, matching
from tests import match_ref as M
from tests import valce_ref as R
from tests.test_gpu_match_bounds import point_indices
from tests.test_gpu_match_exact import probe, tie_pairs

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
KS = [1, 95, 96, 97, 160, 192, 480]
NPTS = [1, 127, 128, 129, 200000]
MODES = ['short', 'long', 'repeat', 'none']


def cases(k):
    """(c, n_pts, mode, label int64, classes) per K: both widths, and across K every n_pts / mode / dtype / classes"""
    i = KS.index(k)
    return [(c, NPTS[(2 * i + j) % 5], MODES[(i + j) % 4], (i + j) % 2 == 1, k if j == 0 else max(1, (2 * k) // 3))
            for j, c in enumerate((512, 768))]


def match_ce(feat, inv, text, label, classes, ignore=R.IGNORE, want=True):
    """one osb_match_ce into prefilled buffers: (scores, pred, loss, areas, bad)"""
    n_pts = inv.shape[0] if inv is not None else feat.shape[0]
    k = text.shape[0]
    scores = torch.full((n_pts, k), float('nan'), dtype=torch.float16, device=DEV) if want else None
    pred = torch.full((n_pts,), -7, dtype=torch.int64, device=DEV) if want else None
    loss = torch.full((1,), 1234.0, dtype=torch.float16, device=DEV)
    areas = torch.zeros((3, classes), dtype=torch.int64, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = torch.full((max(1, 2 * ((n_pts + 127) // 128)),), float('nan'), dtype=torch.float64, device=DEV)
    C.call('osb_match_ce', C.ptr(feat), int(feat.dtype == torch.float16), feat.shape[0], feat.shape[1], C.ptr(inv), n_pts,
           C.ptr(text), k, C.ptr(label), int(label.dtype == torch.int64), ignore, classes, C.ptr(scores), C.ptr(pred),
           C.ptr(loss), C.ptr(areas), C.ptr(bad), C.ptr(ws), 8 * ws.numel(), C.stream_ptr())
    return scores, pred, loss, areas, bad


def labels(n, k, g, dtype):
    y = torch.randint(0, k, (n,), generator=g)
    y[torch.rand(n, generator=g) < 0.15] = R.IGNORE
    return y.to(dtype).to(DEV)


def features(n, c, g):
    return (torch.randn(n, c, generator=g) * (0.5 + 3 * torch.rand(n, 1, generator=g))).to(DEV)


def check_counts(areas, pred, y, classes, k):
    got, bad = R.device_counts(pred.cpu().numpy(), y.cpu().numpy(), classes, k)
    assert np.array_equal(areas.cpu().numpy(), got)
    if bad == 0 and classes > 1:        # histc(bins=1, min=0, max=0) counts over the data's own range instead
        i, u, t = R.intersection_and_union(pred.cpu(), y.cpu().long(), classes)
        a = areas.cpu()
        assert torch.equal(a[0].float(), i) and torch.equal(a[2].float(), t) and torch.equal((a[1] + a[2] - a[0]).float(), u)
    return bad


def check_rows(feat, inv, text, s, y, rows):
    """logp[y] of each row in ``rows`` through the loss of a scene where only that row is labelled"""
    k = text.shape[0]
    sc = s.double().cpu().numpy()
    yc = y.long().cpu().numpy()
    idx = np.array([r for r in rows if yc[r] != R.IGNORE and 0 <= yc[r] < k], dtype=np.int64)
    if len(idx) == 0:
        return
    t = R.logp_at_label(sc[idx], yc[idx])
    fp32 = R.logp_bound(sc[idx], yc[idx])
    half = 0.5 * R.ulp16(np.abs(t) + fp32)
    got = np.empty(len(idx))
    for j, r in enumerate(idx):
        one = torch.full_like(y, R.IGNORE)
        one[r] = y[r]
        _, _, loss, _, _ = match_ce(feat, inv, text, one, 1, want=False)
        got[j] = -float(loss)
    assert np.all(np.abs(got - t) <= fp32 + half), np.max(np.abs(got - t) - fp32 - half)
    tight = fp32 <= 0.5 * R.ulp16(t)
    t16 = t.astype(np.float16).astype(np.float64)
    assert np.all(np.abs(got - t16)[tight] <= R.ulp16(t16)[tight])
    # torch CUDA's log_softmax on the same scores, held to the same bound
    lt = F.log_softmax(s[torch.from_numpy(idx).to(DEV)], dim=1).double().cpu().numpy()[np.arange(len(idx)), yc[idx]]
    assert np.all(np.abs(lt - t) <= fp32 + half), np.max(np.abs(lt - t) - fp32 - half)


@pytest.mark.parametrize('k', KS)
def test_match_ce_against_scores_torch_and_the_fp64_reference(k):
    for j, (c, n_pts, mode, i64, classes) in enumerate(cases(k)):
        g = torch.Generator().manual_seed(17 * k + j)
        n_vox, inv = point_indices(n_pts, mode, g)
        feat = features(n_vox, c, g)
        if j == 1:
            feat = feat.half()
        text = (torch.randn(k, c, generator=g) / math.sqrt(c)).half().to(DEV)
        y = labels(n_pts, k, g, torch.int64 if i64 else torch.int32)
        tag = (k, c, n_pts, mode, i64, classes)
        s, pred, loss, areas, bad = match_ce(feat, inv, text, y, classes)
        ref, _, _ = matching._scores(feat, inv, text, normalize=False)
        assert torch.equal(s.view(torch.int16), ref.view(torch.int16)), tag
        assert torch.equal(pred, s.max(1)[1]), tag
        assert int(bad) == 0 and check_counts(areas, pred, y, classes, k) == 0, tag
        # the scene loss against the fp64 mean of the reference terms and against torch's cross-entropy
        sc, yc = s.double().cpu().numpy(), y.long().cpu().numpy()
        lab = yc != R.IGNORE
        t = R.logp_at_label(sc[lab], yc[lab])
        rb = R.logp_bound(sc[lab], yc[lab]) + 0.5 * R.ulp16(np.abs(t))
        v, _, terms = R.scene_loss(t, yc[lab])
        if len(terms):
            lb = R.loss_bound(terms, rb)
            assert abs(float(loss) - v) <= lb, (tag, float(loss), v, lb)
            tl = float(F.cross_entropy(s, y.long(), ignore_index=R.IGNORE))
            assert abs(float(loss) - tl) <= 2 * lb, (tag, float(loss), tl, lb)
        else:
            assert math.isnan(float(loss))
        # per-row log-probabilities: the first rows, rows across the 128-row block edges, the last rows
        rows = sorted({r for r in list(range(6)) + [127, 128, 129, n_pts // 2, n_pts - 2, n_pts - 1] if 0 <= r < n_pts})
        check_rows(feat, inv, text, s, y, rows)
        # bit-identical rerun
        again = match_ce(feat, inv, text, y, classes)
        for a, b in zip((s, pred, loss, areas, bad), again):
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a,
                               b.view(torch.int16) if b.dtype == torch.float16 else b), tag


def test_rows_with_one_nan_take_its_index_and_all_ignored_or_empty_scenes_are_nan():
    g = torch.Generator().manual_seed(5)
    k, c = 97, 512
    text = (torch.randn(k, c, generator=g) / math.sqrt(c)).half().to(DEV)
    feat = features(300, c, g)
    feat[7, 11] = float('nan')                               # every score of row 7 is NaN: its first column
    y = labels(300, k, g, torch.int64)
    s, pred, loss, areas, bad = match_ce(feat, None, text, y, k)
    assert int(pred[7]) == 0 and torch.equal(pred[8:], s[8:].max(1)[1]) and torch.equal(pred[:7], s[:7].max(1)[1])
    # exactly one NaN per row: a NaN in text row 100 (the second pass) makes column 100 NaN in every row
    k2 = 160
    text2 = (torch.randn(k2, c, generator=g) / math.sqrt(c)).half().to(DEV)
    text2[100, 5] = float('nan')
    s2, pred2, _, _, _ = match_ce(feat[8:], None, text2, y[8:], k2)
    assert bool(torch.isnan(s2[:, 100]).all()) and int(torch.isnan(s2).sum()) == s2.shape[0]
    want = torch.from_numpy(R.argmax_nan_first(s2.float().cpu().numpy())).to(DEV)
    assert bool((pred2 == 100).all()) and torch.equal(pred2, want) and torch.equal(pred2, s2.max(1)[1])
    # all ignored: NaN loss, zero counts, as torch; no points at all: NaN
    none = torch.full((300,), R.IGNORE, dtype=torch.int32, device=DEV)
    _, _, loss, areas, bad = match_ce(feat[8:], None, text, none[8:], 20)
    assert math.isnan(float(loss)) and int(areas.abs().sum()) == 0 and int(bad) == 0
    assert torch.isnan(F.cross_entropy(s[8:], none[8:].long(), ignore_index=R.IGNORE))
    empty = torch.empty(0, dtype=torch.int64, device=DEV)
    _, _, loss, areas, _ = match_ce(feat, empty, text, empty, 20, want=False)
    assert math.isnan(float(loss)) and int(areas.abs().sum()) == 0


def test_bad_labels_are_dropped_counted_and_reported_by_the_meter():
    g = torch.Generator().manual_seed(9)
    k, c, n = 20, 768, 5000
    text = (torch.randn(k, c, generator=g) / math.sqrt(c)).half().to(DEV)
    feat = features(n, c, g)
    y = labels(n, k, g, torch.int64)
    planted = torch.tensor([3, 400, 4999])
    y[planted.to(DEV)] = torch.tensor([k, -1, 1000], device=DEV)
    s, pred, loss, areas, bad = match_ce(feat, None, text, y, k)
    assert int(bad) == 3
    assert check_counts(areas, pred, y, k, k) == 3
    keep = torch.ones(n, dtype=torch.bool)
    keep[planted] = False
    keep = keep.to(DEV)
    _, _, loss_ok, areas_ok, _ = match_ce(feat[keep], None, text, y[keep], k)
    assert torch.equal(areas, areas_ok) and torch.equal(loss.view(torch.int16), loss_ok.view(torch.int16))
    meter = distill.DeviceValidation(text, k)
    good = labels(n, k, g, torch.int64)
    for lab in (good, good, y, good, y):
        meter.add(feat, None, lab)
    with pytest.raises(IndexError, match='scene 2 '):
        meter.end()


@pytest.mark.parametrize('k', [96, 192, 480])
def test_exact_probes_scores_pass_edge_ties_and_counts(k):
    for j, (c, kind) in enumerate([(512, 'f32'), (768, 'f16')]):
        n_pts, mode = (20000, 'long') if j == 0 else (129, 'repeat')
        g = torch.Generator().manual_seed(3 * k + j)
        feat, a, inv, t, n_pl = probe(k, c, n_pts, mode, kind, g)
        ai = a[inv] if inv is not None else a
        assert M.exact_budget_bits(ai, t) < 24
        ref = M.fp16_rn(ai @ t.double().t())
        y = labels(n_pts, k, g, torch.int32)
        s, pred, loss, areas, bad = match_ce(feat, inv, t, y, k)
        exact = (s.view(torch.int16) == ref.view(torch.int16)) | ((s == 0) & (ref == 0))
        assert bool(exact.all()), (k, kind)
        assert torch.equal(pred, ref.float().cpu().max(1)[1].to(DEV)), (k, kind)       # no NaN: the first maximum
        m = min(n_pts, n_pl, len(tie_pairs(k)))
        assert pred[:m].tolist() == [p[0] for p in tie_pairs(k)][:m], (k, kind)
        assert int(bad) == 0 and check_counts(areas, pred, y, k, k) == 0


def test_device_validation_equals_the_torch_tail_on_engine_outputs():
    """FusedMinkUNet(model, batch_stats=True) forwards of config1_50k scenes (MinkUNet18A), the same outputs fed to the
    restated torch tail of validate() and to DeviceValidation; the torch tail's scores are osb_match_scores' (bit-identical
    to the meter's product), so both see the same scores."""
    from openscene_b200 import engine, synth
    torch.cuda.set_device(0)
    k = classes = 20
    text = torch.from_numpy(synth.text_embeddings(k)).to(DEV)
    model = synth.build_model('MinkUNet18A', 768, seed=0).train().to(DEV)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    meter = distill.DeviceValidation(text, classes)
    scenes, bounds = [], []
    for seed in range(4):
        coords = torch.from_numpy(synth.scene('config1_50k', seed=seed)).to(DEV)
        g = torch.Generator().manual_seed(seed)
        n_vox = coords.shape[0]
        inv = torch.cat([torch.randperm(n_vox, generator=g), torch.randint(0, n_vox, (n_vox // 2,), generator=g)])
        band = (coords[:, 3].float() / (coords[:, 3].max().float() + 1)).cpu()
        label = (band[inv] * classes).long().clamp(max=classes - 1)
        label[torch.rand(len(inv), generator=g) < 0.15] = R.IGNORE
        feats = torch.rand(n_vox, 3, generator=g).to(DEV)
        with torch.no_grad():
            output = eng(coords, feats)
        meter.add(output, inv, label)
        # the torch tail, one scene
        lab = label.to(DEV)
        scores, _, _ = matching._scores(output, inv.to(DEV), text, normalize=False)
        loss = F.cross_entropy(scores, lab, ignore_index=R.IGNORE)
        pred = torch.max(scores, 1)[1]
        i, u, t = R.intersection_and_union(pred.cpu(), lab.cpu(), classes)
        i, u, t = i.cuda(), u.cuda(), t.cuda()
        scenes.append((loss.item(), i.cpu().numpy(), u.cpu().numpy(), t.cpu().numpy()))
        sc, yc = scores.double().cpu().numpy(), label.numpy()
        m = yc != R.IGNORE
        tt = R.logp_at_label(sc[m], yc[m])
        bounds.append(2 * R.loss_bound(-tt, R.logp_bound(sc[m], yc[m]) + 0.5 * R.ulp16(np.abs(tt))))
    got = meter.end(weight=1)
    want = R.validate_tail(scenes, batch_size=1)
    assert R.same(got[1:], want[1:]), (got, want)
    assert abs(got[0] - want[0]) <= float(np.mean(bounds)), (got[0], want[0])
    meter.begin()
    assert meter.n == 0
