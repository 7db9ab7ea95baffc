"""Open-vocabulary matching on libosb200 (csrc/match.cu): the three ``feature_type`` branches of
``run/evaluate.py:288-323`` with the same arguments and results (fp16 scores [N_pts, K], int64 labels),
computed in one pass per product without materialising ``predictions[inds_reverse]``."""
import torch

from . import _cabi as C


def _scores(feat, inds_reverse, text, normalize, want_scores=True, want_smax=False):
    C.require_cuda(feat, 'features')
    feat = feat.contiguous()
    text = text.to(device=feat.device, dtype=torch.float16).contiguous()
    is_f16 = feat.dtype == torch.float16
    if not is_f16 and feat.dtype != torch.float32:
        feat = feat.float()
    n_vox, c = feat.shape
    k = text.shape[0]
    assert text.shape[1] == c, f"text embeddings have width {text.shape[1]}, features {c}"
    if inds_reverse is not None:
        inds_reverse = inds_reverse.to(device=feat.device, dtype=torch.int64).contiguous()
        n_pts = inds_reverse.shape[0]
    else:
        n_pts = n_vox
    with torch.cuda.device(feat.device):
        scores = torch.empty((n_pts, k), dtype=torch.float16, device=feat.device) if want_scores else None
        label = torch.empty(n_pts, dtype=torch.int64, device=feat.device)
        smax = torch.empty(n_pts, dtype=torch.float32, device=feat.device) if want_smax else None
        C.call('osb_match_scores', C.ptr(feat), int(is_f16), n_vox, c, C.ptr(inds_reverse), n_pts, C.ptr(text), k,
               int(normalize), C.ptr(scores), C.ptr(label), C.ptr(smax), C.stream_ptr())
    return scores, label, smax


def match_distill(predictions, inds_reverse, text_features):
    """evaluate.py:288-292: ``pred = predictions[inds_reverse].half() @ text.t(); label = argmax``."""
    s, l, _ = _scores(predictions, inds_reverse, text_features, normalize=False)
    return s, l


def match_fusion(feat_3d, inds_reverse, text_features):
    """evaluate.py:293-296 (fused 2-D features, fp16)."""
    s, l, _ = _scores(feat_3d, inds_reverse, text_features, normalize=False)
    return s, l


def match_ensemble(predictions, feat_3d, inds_reverse, text_features, return_features=False):
    """evaluate.py:302-323: cosine scores of both feature sets, per-point winner, final product.

    Returns (pred fp16 [N_pts,K], label int64 [N_pts], feat_ensemble fp16 [N_pts,C] or None, mask bool)."""
    feat_3d = feat_3d.to(predictions.device)
    if feat_3d.dtype != torch.float16:
        feat_3d = feat_3d.half()
    _, _, smax2d = _scores(feat_3d, inds_reverse, text_features, normalize=True, want_scores=False, want_smax=True)
    _, _, smax3d = _scores(predictions, inds_reverse, text_features, normalize=True, want_scores=False, want_smax=True)
    predictions = predictions.contiguous().float()
    feat_3d = feat_3d.contiguous()
    text = text_features.to(device=predictions.device, dtype=torch.float16).contiguous()
    n_vox, c = predictions.shape
    inv = inds_reverse.to(device=predictions.device, dtype=torch.int64).contiguous() if inds_reverse is not None else None
    n_pts = inv.shape[0] if inv is not None else n_vox
    k = text.shape[0]
    with torch.cuda.device(predictions.device):
        scores = torch.empty((n_pts, k), dtype=torch.float16, device=predictions.device)
        label = torch.empty(n_pts, dtype=torch.int64, device=predictions.device)
        fe = torch.empty((n_pts, c), dtype=torch.float16, device=predictions.device) if return_features else None
        C.call('osb_match_ensemble', C.ptr(predictions), C.ptr(feat_3d), n_vox, c, C.ptr(inv), n_pts, C.ptr(smax3d),
               C.ptr(smax2d), C.ptr(text), k, C.ptr(scores), C.ptr(label), C.ptr(fe), C.stream_ptr())
    return scores, label, fe, smax3d < smax2d


def _topk(feat, inds_reverse, text, k, normalize, want_scores, want_smax=False):
    """one osb_match_topk: (scores fp16 [N_pts, k] | None, labels int64 [N_pts, k], smax fp32 [N_pts] | None)"""
    C.require_cuda(feat, 'features')
    feat = feat.contiguous()
    if feat.dtype not in (torch.float16, torch.float32):
        feat = feat.float()
    text = text.to(device=feat.device, dtype=torch.float16).contiguous()
    n_vox, c = feat.shape
    assert text.shape[1] == c, f"text embeddings have width {text.shape[1]}, features {c}"
    inv = inds_reverse.to(device=feat.device, dtype=torch.int64).contiguous() if inds_reverse is not None else None
    n_pts = inv.shape[0] if inv is not None else n_vox
    with torch.cuda.device(feat.device):
        scores = torch.empty((n_pts, k), dtype=torch.float16, device=feat.device) if want_scores else None
        label = torch.empty((n_pts, k), dtype=torch.int64, device=feat.device)
        smax = torch.empty(n_pts, dtype=torch.float32, device=feat.device) if want_smax else None
        C.call('osb_match_topk', C.ptr(feat), int(feat.dtype == torch.float16), n_vox, c, C.ptr(inv), n_pts, C.ptr(text),
               text.shape[0], int(normalize), k, C.ptr(scores), C.ptr(label), C.ptr(smax), C.stream_ptr())
    return scores, label, smax


def match_topk(feat, inds_reverse, text_features, k=1, normalize=False, want_scores=True):
    """The distill / fusion branches of evaluate.py:288-296 for a label set of any size (up to 2^20 rows): the k best
    columns of ``feat[inds_reverse].half() @ text.t()`` per point, best first, without the [N_pts, K] scores.  NaN ranks
    first, equal scores go to the lower column (DESIGN.md, "Top-k match contract").  ``normalize`` applies
    x / (|x| + 1e-5) first.  Returns (scores fp16 [N_pts, k] or None, labels int64 [N_pts, k]); labels[:, 0] is the
    prediction."""
    s, l, _ = _topk(feat, inds_reverse, text_features, k, normalize, want_scores)
    return s, l


def match_ensemble_topk(predictions, feat_3d, inds_reverse, text_features, k=1, return_features=False):
    """evaluate.py:302-323 for a label set of any size: two streaming passes for the normalised row maxima of both feature
    sets, the per-point winner, and the top-k of the final product on it.  Returns (scores fp16 [N_pts, k], labels int64
    [N_pts, k], feat_ensemble fp16 [N_pts, C] or None, mask bool = smax3d < smax2d)."""
    feat_3d = feat_3d.to(predictions.device)
    if feat_3d.dtype != torch.float16:
        feat_3d = feat_3d.half()
    _, _, smax2d = _topk(feat_3d, inds_reverse, text_features, 1, True, False, want_smax=True)
    _, _, smax3d = _topk(predictions, inds_reverse, text_features, 1, True, False, want_smax=True)
    predictions = predictions.contiguous().float()
    feat_3d = feat_3d.contiguous()
    text = text_features.to(device=predictions.device, dtype=torch.float16).contiguous()
    n_vox, c = predictions.shape
    inv = inds_reverse.to(device=predictions.device, dtype=torch.int64).contiguous() if inds_reverse is not None else None
    n_pts = inv.shape[0] if inv is not None else n_vox
    with torch.cuda.device(predictions.device):
        scores = torch.empty((n_pts, k), dtype=torch.float16, device=predictions.device)
        label = torch.empty((n_pts, k), dtype=torch.int64, device=predictions.device)
        fe = torch.empty((n_pts, c), dtype=torch.float16, device=predictions.device) if return_features else None
        C.call('osb_match_ensemble_topk', C.ptr(predictions), C.ptr(feat_3d), n_vox, c, C.ptr(inv), n_pts, C.ptr(smax3d),
               C.ptr(smax2d), C.ptr(text), text.shape[0], k, C.ptr(scores), C.ptr(label), C.ptr(fe), C.stream_ptr())
    return scores, label, fe, smax3d < smax2d
