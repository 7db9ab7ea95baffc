"""CPU restatement of the test-time repeat loops of ``run/evaluate.py:385-425`` and ``run/eval_mink.py:167-216``, with
the same torch CPU operations in the same order: per-repeat concatenation of the scene score matrices, ``pred + store``
(store starting at the Python float 0.0), ``.float().max(1)[1]``, ``mapper``, the no-feature override and the metric
(``oracle.metric_ref``).  Test infrastructure: the product (``openscene_b200.repeat_eval``) never imports it."""
import torch

from oracle import metric_ref


def evaluate_py(repeats, gts, num_classes, mapper=None, masks=None):
    """evaluate.py with ``test_repeats > 1``.

    repeats  list over repeats of lists over scenes of fp16 CPU scores [N_pts, K] (the ``pred`` of each scene)
    gts      list over scenes of int64 labels [N_pts]
    masks    None, or list over repeats of lists over scenes of bool [N_pts] (``mask[inds_reverse]``)
    Returns a list over repeats of dicts: store, pred_logit, store_logit (mapped, overridden), cur_iou, acc_iou."""
    gt = torch.cat(gts)
    mapper = None if mapper is None else torch.as_tensor(mapper)
    store = 0.0
    out = []
    for r, preds in enumerate(repeats):
        pred = torch.cat(preds)
        pred_logit = pred.float().max(1)[1]
        if mapper is not None:
            pred_logit = mapper[pred_logit]
        if masks is not None:
            mask = torch.cat(masks[r])
            pred_logit[~mask] = 256
        store = pred + store
        store_logit = store.float().max(1)[1]
        if mapper is not None:
            store_logit = mapper[store_logit]
        if masks is not None:
            store_logit[~mask] = 256
        out.append(dict(store=store, pred_logit=pred_logit, store_logit=store_logit,
                        cur_iou=metric_ref.mean_iou(pred_logit.numpy(), gt.numpy(), num_classes)[0],
                        acc_iou=metric_ref.mean_iou(store_logit.numpy(), gt.numpy(), num_classes)[0]))
    return out


def eval_mink_py(repeats, gts, num_classes, nuscenes=False):
    """eval_mink.py with ``test_repeats > 1``: repeats = list over repeats of lists over scenes of fp32 CPU
    ``predictions[inds_reverse]``; with ``nuscenes`` only the points with ``label != 255`` are kept, as there."""
    store = 0.0
    out = []
    for preds in repeats:
        ps, gs = [], []
        for p, label in zip(preds, gts):
            if nuscenes:
                label_mask = label != 255
                label, p = label[label_mask], p[label_mask]
            ps.append(p)
            gs.append(label)
        gt, pred = torch.cat(gs), torch.cat(ps)
        cur = pred.max(1)[1]
        store = pred + store
        acc = store.max(1)[1]
        out.append(dict(store=store, pred_logit=cur, store_logit=acc,
                        cur_iou=metric_ref.mean_iou(cur.numpy(), gt.numpy(), num_classes)[0],
                        acc_iou=metric_ref.mean_iou(acc.numpy(), gt.numpy(), num_classes)[0]))
    return out


def same_bits(a, b):
    """Equal bit patterns, except that any NaN equals any NaN (payloads are not part of the contract)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    itype = torch.int16 if a.dtype == torch.float16 else torch.int32
    return torch.equal(a[~na].view(itype), b[~nb].view(itype))
