"""The test-time repeat vote on the GPU: the vote epilogue of the tensor-core match (osb_match_vote /
osb_match_ensemble_vote) against the separate route (osb_match_scores + osb_vote_accumulate) and against the reference's
CPU loop fed the same scores (tests/vote_oracle.py), bit for bit; the fp32 logits path; and ``RepeatVote`` end to end on
re-voxelised scenes through the eval engine."""
import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import matching, synth
from tests.vote_oracle import eval_mink_py, evaluate_py, same_bits

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _feats(n, c, seed, f16):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(n, c, generator=g) * (0.2 + torch.rand(n, 1, generator=g))
    f[:4] *= 1e5          # fp16 operands overflow: inf / NaN scores
    f[4:8] *= 300         # finite scores that overflow the fp16 store within a few repeats
    return f.half() if f16 else f


def _vote_fused(feat, inv, text, store, scores=None, normalize=0):
    n_pts = inv.shape[0] if inv is not None else feat.shape[0]
    lc = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    la = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    C.call('osb_match_vote', C.ptr(feat), int(feat.dtype == torch.float16), feat.shape[0], feat.shape[1], C.ptr(inv), n_pts,
           C.ptr(text), text.shape[0], normalize, C.ptr(scores), C.ptr(store), C.ptr(lc), C.ptr(la), C.stream_ptr())
    return lc, la


def _vote_separate(scores, store, src_is_f16=True):
    n_pts, k = scores.shape
    lc = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    la = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    C.call('osb_vote_accumulate', C.ptr(scores), int(src_is_f16), n_pts, None, n_pts, k, C.ptr(store), C.ptr(lc), C.ptr(la),
           C.stream_ptr())
    return lc, la


def _check_against_separate_and_oracle(run_fused, run_scores, n_pts, k, repeats=5):
    """run_fused(r, store) -> (label_cur, label_acc); run_scores(r) -> this repeat's fp16 scores (the existing kernels)"""
    st_f = torch.zeros((n_pts, k), dtype=torch.float16, device=DEV)
    st_s = torch.zeros_like(st_f)
    preds = []
    for r in range(repeats):
        lc, la = run_fused(r, st_f)
        s = run_scores(r)
        lc2, la2 = _vote_separate(s, st_s)
        preds.append([s.cpu()])
        ref = evaluate_py(preds, [torch.zeros(n_pts, dtype=torch.int64)], k)[-1]
        assert torch.equal(st_f.view(torch.int16), st_s.view(torch.int16)), f"repeat {r}: fused and separate stores differ"
        assert same_bits(st_f.cpu(), ref['store']), f"repeat {r}: store differs from the CPU `pred + store`"
        assert torch.equal(lc, lc2) and torch.equal(la, la2)
        assert torch.equal(lc.cpu(), ref['pred_logit']) and torch.equal(la.cpu(), ref['store_logit'])
    return st_f


@pytest.mark.parametrize('inds', [True, False])
@pytest.mark.parametrize('f16', [False, True])
@pytest.mark.parametrize('c', [512, 768])
@pytest.mark.parametrize('k', [16, 20, 21, 40, 80, 160])
def test_fused_vote_equals_separate_route_and_oracle(k, c, f16, inds):
    n_vox = 1500
    n_pts = 2037 if inds else n_vox          # not a multiple of the 128-point tile
    text = torch.from_numpy(synth.text_embeddings(k, c)).to(DEV)
    feats = [_feats(n_vox, c, 10 * k + r, f16).to(DEV) for r in range(5)]
    invs = [torch.randint(0, n_vox, (n_pts,), generator=torch.Generator().manual_seed(r)).to(DEV) if inds else None
            for r in range(5)]
    store = _check_against_separate_and_oracle(
        lambda r, st: _vote_fused(feats[r], invs[r], text, st),
        lambda r: matching._scores(feats[r], invs[r], text, normalize=False)[0], n_pts, k)
    finite = torch.isfinite(store.float())
    assert (~finite).any() and finite.any()          # the overflow rows reached the store


def test_scores_output_is_bit_identical_to_match_scores():
    for k, c in ((20, 768), (160, 512)):
        text = torch.from_numpy(synth.text_embeddings(k, c)).to(DEV)
        f = _feats(1300, c, 7, False).to(DEV)
        inv = torch.randint(0, 1300, (3001,), generator=torch.Generator().manual_seed(3)).to(DEV)
        for normalize in (0, 1):
            s = torch.empty((3001, k), dtype=torch.float16, device=DEV)
            _vote_fused(f, inv, text, torch.zeros((3001, k), dtype=torch.float16, device=DEV), scores=s, normalize=normalize)
            ref = matching._scores(f, inv, text, normalize=bool(normalize))[0]
            assert torch.equal(s.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize('k,c', [(20, 768), (160, 768), (21, 512)])
def test_ensemble_vote(k, c):
    n_vox, n_pts = 1400, 2111
    text = torch.from_numpy(synth.text_embeddings(k, c)).to(DEV)
    f3 = [_feats(n_vox, c, r, False).to(DEV) for r in range(5)]
    f2 = [_feats(n_vox, c, 100 + r, False).clamp(-5, 5).half().to(DEV) for r in range(5)]
    invs = [torch.randint(0, n_vox, (n_pts,), generator=torch.Generator().manual_seed(r)).to(DEV) for r in range(5)]

    def smax(r):
        _, _, s2 = matching._scores(f2[r], invs[r], text, normalize=True, want_scores=False, want_smax=True)
        _, _, s3 = matching._scores(f3[r], invs[r], text, normalize=True, want_scores=False, want_smax=True)
        return s3, s2

    def fused(r, st):
        s3, s2 = smax(r)
        lc = torch.empty(n_pts, dtype=torch.int64, device=DEV)
        la = torch.empty(n_pts, dtype=torch.int64, device=DEV)
        C.call('osb_match_ensemble_vote', C.ptr(f3[r]), C.ptr(f2[r]), n_vox, c, C.ptr(invs[r]), n_pts, C.ptr(s3), C.ptr(s2),
               C.ptr(text), k, None, C.ptr(st), C.ptr(lc), C.ptr(la), C.stream_ptr())
        return lc, la

    def scores(r):
        s, _, _, _ = matching.match_ensemble(f3[r], f2[r], invs[r], text)
        return s

    _check_against_separate_and_oracle(fused, scores, n_pts, k)


def test_fp32_logits_path_equals_cpu_sum():
    from openscene_b200.repeat_eval import RepeatVote
    g = torch.Generator().manual_seed(0)
    vote = RepeatVote(20, store_dtype=torch.float32)
    n_vox, n_pts = [900, 1300], [1500, 2222]
    gts = [torch.randint(0, 20, (n,), generator=g) for n in n_pts]
    for s in range(2):
        gts[s][::7] = 255
    preds = []
    for r in range(4):
        vote.begin_repeat()
        rep = []
        for s in range(2):
            logits = torch.randn(n_vox[s], 20, generator=g) * 4
            logits[3] = float('nan')
            logits[5, 7] = float('inf')
            inv = torch.randint(0, n_vox[s], (n_pts[s],), generator=g)
            lc = vote.add_logits(s, logits.to(DEV), inv.to(DEV), gt=gts[s].to(DEV))
            rep.append(logits[inv])
            assert torch.equal(lc.cpu(), logits[inv].max(1)[1])
        preds.append(rep)
        cur, acc = vote.end_repeat()
        ref = eval_mink_py(preds, gts, 20)[-1]
        store = torch.cat([vote.scenes[s].store.cpu() for s in range(2)])
        assert same_bits(store, ref['store'])
        assert torch.equal(vote.labels().cpu(), ref['store_logit'])
        assert (cur, acc) == (ref['cur_iou'], ref['acc_iou'])
        # nuScenes: eval_mink keeps only label != 255; the full vote counted on the kept points gives the same numbers
        refn = eval_mink_py(preds, gts, 20, nuscenes=True)[-1]
        assert (cur, acc) == (refn['cur_iou'], refn['acc_iou'])


def test_reproducible_stores():
    k, c = 40, 768
    text = torch.from_numpy(synth.text_embeddings(k, c)).to(DEV)
    f = _feats(3000, c, 1, False).to(DEV)
    inv = torch.randint(0, 3000, (5000,), generator=torch.Generator().manual_seed(1)).to(DEV)
    runs = []
    for _ in range(2):
        st = torch.zeros((5000, k), dtype=torch.float16, device=DEV)
        for _ in range(3):
            _vote_fused(f, inv, text, st)
        runs.append(st)
    assert torch.equal(runs[0].view(torch.int16), runs[1].view(torch.int16))


# ------------------------------------------------------------------------------------------------------ end to end
def _scene_labels(pts, k):
    """ground truth from the geometry: height bands x slabs, 5 % unlabelled (255)"""
    p = torch.from_numpy(pts)
    lab = ((p[:, 2] * 5).long() * 3 + (p[:, 0] * 4).long()) % k
    lab[torch.arange(len(p)) % 20 == 0] = 255
    return lab


def _run_e2e(k=20, num_classes=20, mapper=None, nofeat=False, n_scenes=3, repeats=3):
    from openscene_b200 import engine
    from openscene_b200.repeat_eval import RepeatVote
    from openscene_b200.voxelize import Voxelizer, voxelize_points
    torch.manual_seed(0)
    model = synth.build_model('MinkUNet18A', 768, seed=0).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    text = torch.from_numpy(synth.text_embeddings(k, 768)).to(DEV)
    scenes = [synth.room_points((1.0 + 0.2 * s, 0.8, 0.7), 2, seed=s) for s in range(n_scenes)]
    gts = [_scene_labels(p, num_classes) for p in scenes]
    vox = Voxelizer(voxel_size=0.02, use_augmentation=True, scale_augmentation_bound=(0.9, 1.1),
                    rotation_augmentation_bound=((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi)))
    np.random.seed(0)
    vote = RepeatVote(num_classes, mapper=mapper)
    ours, preds, cublas, masks = [], [], [], []
    for r in range(repeats):
        vote.begin_repeat()
        rep, repc, repm = [], [], []
        for s, pts in enumerate(scenes):
            M_v, M_r = vox.get_transformation_matrix()
            cv, inds, inv, _ = voxelize_points(torch.from_numpy(pts).to(DEV), M_r @ M_v)
            c4 = torch.zeros((cv.shape[0], 4), dtype=torch.int32, device=DEV)
            c4[:, 1:] = cv
            with torch.no_grad():
                out = eng(c4, torch.ones(cv.shape[0], 3, device=DEV))
            m = (torch.arange(len(pts), device=DEV) + r) % 11 != 0 if nofeat else None
            vote.match_distill(s, out, inv, text, gt=gts[s].to(DEV), nofeat=m)
            rep.append(matching.match_distill(out, inv, text)[0].cpu())
            repc.append((out[inv].half() @ text.t()).cpu())
            repm.append(m.cpu() if m is not None else None)
        ours.append(vote.end_repeat())
        preds.append(rep)
        cublas.append(repc)
        masks.append(repm)
    return vote, ours, preds, cublas, gts, (masks if nofeat else None)


def _check_e2e(vote, ours, preds, cublas, gts, masks, num_classes, mapper=None):
    ref = evaluate_py(preds, gts, num_classes, mapper=mapper, masks=masks)
    for r, (cur, acc) in enumerate(ours):
        assert (cur, acc) == (ref[r]['cur_iou'], ref[r]['acc_iou']), f"repeat {r}"
    store = torch.cat([vote.scenes[s].store.cpu() for s in range(len(gts))])
    assert same_bits(store, ref[-1]['store'])
    # against the reference's own cuBLAS product: the accumulated labels agree wherever the top-two gap is clear
    cb = evaluate_py(cublas, gts, num_classes, mapper=mapper)[-1]['store'].float()
    lab = vote.labels().cpu()
    top2 = cb.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-3 * top2[:, 0].abs()
    cb_lab = cb.max(1)[1]
    assert (lab == cb_lab).float().mean() >= 0.999
    assert torch.equal(lab[clear], cb_lab[clear])


def test_end_to_end_three_scenes_three_repeats():
    res = _run_e2e()
    _check_e2e(*res, num_classes=20)


def test_end_to_end_nuscenes_mapper_and_subset():
    mapper = torch.arange(20) % 16
    vote, ours, preds, cublas, gts, _ = _run_e2e(num_classes=16, mapper=mapper)
    _check_e2e(vote, ours, preds, cublas, gts, None, 16, mapper=mapper)
    # evaluate.py's nuScenes branch keeps only label != 255 before storing: the same IoUs on the subset
    keep = [g != 255 for g in gts]
    sub = evaluate_py([[p[m] for p, m in zip(rep, keep)] for rep in preds], [g[m] for g, m in zip(gts, keep)], 16,
                      mapper=mapper)
    for r, (cur, acc) in enumerate(ours):
        assert (cur, acc) == (sub[r]['cur_iou'], sub[r]['acc_iou'])


def test_end_to_end_mark_no_feature_to_unknown():
    vote, ours, preds, cublas, gts, masks = _run_e2e(nofeat=True)
    _check_e2e(vote, ours, preds, cublas, gts, masks, 20)


_SIMT_CHILD = r'''
import sys
sys.path.insert(0, sys.argv[1])
import torch
from openscene_b200 import _cabi as C
from openscene_b200 import matching, synth
from tests.test_gpu_repeat_vote import DEV, _feats, _vote_fused
from tests.vote_oracle import evaluate_py, same_bits
k, c, n_pts = 21, 768, 1999
text = torch.from_numpy(synth.text_embeddings(k, c)).to(DEV)
st = torch.zeros((n_pts, k), dtype=torch.float16, device=DEV)
preds = []
for r in range(3):
    f = _feats(1200, c, r, False).to(DEV)
    inv = torch.randint(0, 1200, (n_pts,), generator=torch.Generator().manual_seed(r)).to(DEV)
    lc, la = _vote_fused(f, inv, text, st)
    preds.append([matching._scores(f, inv, text, normalize=False)[0].cpu()])
    ref = evaluate_py(preds, [torch.zeros(n_pts, dtype=torch.int64)], k)[-1]
    assert same_bits(st.cpu(), ref['store']), r
    assert torch.equal(lc.cpu(), ref['pred_logit']) and torch.equal(la.cpu(), ref['store_logit']), r
print('SIMT_OK')
'''


def test_simt_route_of_the_match_vote():
    """OSB_MATCH_SIMT=1 (read once per process, hence a child): CUDA-core scores into scratch, then k_vote_accumulate"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, '-c', _SIMT_CHILD, root], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, OSB_MATCH_SIMT='1'))
    assert p.returncode == 0 and 'SIMT_OK' in p.stdout, p.stderr[-3000:]


def test_unaligned_store_takes_the_two_access_route():
    """an even K with a store that is only 2-byte aligned: the fused vote must not use the paired 4-byte access"""
    k, c, n_pts = 20, 768, 1777
    text = torch.from_numpy(synth.text_embeddings(k, c)).to(DEV)
    flat = torch.zeros(n_pts * k + 1, dtype=torch.float16, device=DEV)
    st_f = flat[1:].view(n_pts, k)
    st_s = torch.zeros((n_pts, k), dtype=torch.float16, device=DEV)
    for r in range(3):
        f = _feats(1200, c, r, False).to(DEV)
        inv = torch.randint(0, 1200, (n_pts,), generator=torch.Generator().manual_seed(r)).to(DEV)
        lc, la = _vote_fused(f, inv, text, st_f)
        lc2, la2 = _vote_separate(matching._scores(f, inv, text, normalize=False)[0], st_s)
        assert torch.equal(st_f.view(torch.int16), st_s.view(torch.int16)) and flat[0].item() == 0
        assert torch.equal(lc, lc2) and torch.equal(la, la2)


@pytest.mark.parametrize('dataset', ['scannet_3d', 'nuscenes_3d'])
def test_documented_binding_reports_a_perfect_vote_as_one(dataset):
    """evaluate.py's binding ``RepeatVote(None, dataset=labelset_name, mapper=mapper)`` on text features of the labelset
    without its appended 'unlabeled': points whose feature is their own class's text row score mIoU 1.0 in every repeat"""
    from openscene_b200.repeat_eval import RepeatVote
    if dataset == 'scannet_3d':
        k, mapper = 20, None
    else:
        k, mapper = 43, torch.arange(43) * 16 // 43         # detailed nuScenes names -> 16 classes
    text = torch.from_numpy(synth.text_embeddings(k, 768)).to(DEV)
    vote = RepeatVote(None, dataset=dataset, mapper=mapper)
    g = torch.Generator().manual_seed(5)
    n_vox, n_pts = 700, 1100
    cls = torch.arange(n_vox) % k                            # voxel v holds class v % k
    pt_cls = [torch.arange(n_pts) % k, (torch.arange(n_pts) * 7) % k]        # every class present in every scene
    for r in range(2):
        vote.begin_repeat()
        for s in range(2):
            # a new voxelisation per repeat: each point lands in a random voxel of its own class
            inv = pt_cls[s] + k * torch.randint(0, n_vox // k, (n_pts,), generator=g)
            gt = pt_cls[s] if mapper is None else mapper[pt_cls[s]]
            gt = gt.clone()
            gt[::13] = 255
            vote.match_distill(s, text[cls.to(DEV)].float(), inv.to(DEV), text, gt=gt.to(DEV))
        cur, acc = vote.end_repeat()
        assert cur == 1.0 and acc == 1.0, (cur, acc)
