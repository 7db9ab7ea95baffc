"""Segmentation metrics accumulated on the GPU (SURVEY.md 8f rank 4) behind the reference's function names:
``confusion_matrix`` / ``get_iou`` / ``evaluate`` (``util/metric.py``) and ``intersectionAndUnionGPU``
(``util/util.py:132-145``, which copies to the host for ``torch.histc``).  Counting runs in csrc/metric.cu."""
import numpy as np
import torch

from . import _cabi as C

UNKNOWN_ID = 255
NO_FEATURE_ID = 256

# len() of the label lists evaluate() picks (util/metric.py:47-60, dataset/label_constants.py); order matters: first match wins
_DATASET_CLASSES = (('scannet_3d', 20), ('matterport_3d_40', 40), ('matterport_3d_80', 80), ('matterport_3d_160', 160),
                    ('matterport_3d', 21), ('nuscenes_3d', 16))


def _labels(x, device):
    t = torch.as_tensor(x)
    if t.dtype not in (torch.int32, torch.int64):
        t = t.long()
    return t.to(device).contiguous().view(-1)


class ConfusionMeter:
    """Device-resident (C+1)x(C+1) confusion matrix; ``update`` never synchronises, so a validation loop can call it
    per batch and read the result once."""

    def __init__(self, num_classes, device='cuda'):
        self.C = num_classes
        self.device = torch.device(device)
        self.full = torch.zeros((num_classes + 1, num_classes + 1), dtype=torch.int64, device=self.device)
        self.bad = torch.zeros(1, dtype=torch.int32, device=self.device)

    def update(self, pred_ids, gt_ids):
        p, g = _labels(pred_ids, self.device), _labels(gt_ids, self.device)
        assert p.shape == g.shape, (p.shape, g.shape)
        if p.dtype != g.dtype:
            p, g = p.long(), g.long()
        with torch.cuda.device(self.device):
            C.call('osb_confusion_accumulate', C.ptr(p), C.ptr(g), int(p.dtype == torch.int64), p.numel(), self.C, UNKNOWN_ID,
                   NO_FEATURE_ID, C.ptr(self.full), C.ptr(self.bad), C.stream_ptr())

    def confusion(self):
        """numpy ulonglong [C,C] as util/metric.py:9-25 returns it.  SYNC."""
        if int(self.bad.item()):
            raise ValueError(f"openscene_b200.metric: {int(self.bad.item())} labels outside 0..{self.C - 1} (gt) / 0..{self.C - 1}, 256 (pred)")
        return self.full[:self.C, :self.C].cpu().numpy().astype(np.ulonglong)

    def evaluate(self):
        """(mean_iou, mean_acc, class_ious) with the reference's conventions (util/metric.py:62-78): classes absent from
        the ground truth are skipped but the mean divides by ALL classes.  SYNC."""
        conf = self.confusion().astype(np.int64)
        gt_count = self.full[:, :self.C].sum(0).cpu().numpy()                  # (gt_ids == i).sum(), 'no feature' rows included
        mean_iou = mean_acc = 0.0
        ious = {}
        for i in range(self.C):
            if gt_count[i] == 0:
                continue
            ious[i] = get_iou(i, conf)
            mean_iou += ious[i][0]
            mean_acc += ious[i][1] / gt_count[i]
        return mean_iou / self.C, mean_acc / self.C, ious


def confusion_matrix(pred_ids, gt_ids, num_classes):
    m = ConfusionMeter(num_classes)
    m.update(pred_ids, gt_ids)
    return m.confusion()


def get_iou(label_id, confusion):
    """util/metric.py:28-41."""
    tp = np.longlong(confusion[label_id, label_id])
    fp = np.longlong(confusion[label_id, :].sum()) - tp
    fn = np.longlong(confusion[:, label_id].sum()) - tp
    denom = tp + fp + fn
    if denom == 0:
        return float('nan')
    return float(tp) / denom, tp, denom


def evaluate(pred_ids, gt_ids, stdout=False, dataset='scannet_3d'):
    """util/metric.py:44-103; returns the mean IoU."""
    for key, n_classes in _DATASET_CLASSES:
        if key in dataset:
            break
    else:
        raise NotImplementedError
    m = ConfusionMeter(n_classes)
    m.update(pred_ids, gt_ids)
    mean_iou, mean_acc, ious = m.evaluate()
    if stdout:
        print_evaluation(int(torch.as_tensor(gt_ids).numel()), mean_iou, mean_acc, ious)
    return mean_iou


def print_evaluation(n_points, mean_iou, mean_acc, ious):
    """The report ``evaluate(..., stdout=True)`` prints (util/metric.py:80-101)."""
    print('evaluating', n_points, 'points...')
    for i, v in ious.items():
        print('class {0:<4d}: {1:>5.3f}   ({2:>6d}/{3:<6d})'.format(i, v[0], int(v[1]), int(v[2])))
    print('Mean IoU', mean_iou)
    print('Mean Acc', mean_acc)


def intersectionAndUnionGPU(output, target, K, ignore_index=255):
    """util/util.py:132-145 without the host round trip: float32 CUDA tensors (area_intersection, area_union,
    area_target).  Unlike the reference it does not overwrite ``output`` where ``target == ignore_index``."""
    assert output.dim() in [1, 2, 3, 4]
    assert output.shape == target.shape
    C.require_cuda(output, 'output')
    o, t = _labels(output, output.device), _labels(target, output.device)
    if o.dtype != t.dtype:
        o, t = o.long(), t.long()
    with torch.cuda.device(output.device):
        areas = torch.zeros((3, K), dtype=torch.int64, device=output.device)
        C.call('osb_intersection_union', C.ptr(o), C.ptr(t), int(o.dtype == torch.int64), o.numel(), K, ignore_index, C.ptr(areas),
               C.stream_ptr())
    inter, a_out, a_tgt = areas[0].float(), areas[1].float(), areas[2].float()
    return inter, a_out + a_tgt - inter, a_tgt
