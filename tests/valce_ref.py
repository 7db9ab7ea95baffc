"""NumPy / fp64 restatement of the validation tail of run/distill.py (:419-446) that ``osb_match_ce`` and
``openscene_b200.distill.DeviceValidation`` compute: the per-row cross-entropy term, the scene loss, the argmax, the
intersection / union / target counts and the host meter replay.  The reference is restated here, not imported."""
import math

import numpy as np
import torch

U = 2.0 ** -24            # fp32 unit roundoff
IGNORE = 255


def ulp16(x):
    """Spacing of fp16 at |x| (the subnormal spacing 2^-24 below 2^-14)."""
    a = np.abs(np.asarray(x, dtype=np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.where(np.isfinite(a), 2.0 ** (np.minimum(e, 15) - 10), np.inf)


def logp_at_label(scores16, y):
    """T = (s_y - m) - log(sum_k exp(s_k - m)) in fp64 from the fp16 scores, per row (rows with y outside [0, K) get NaN)."""
    s = np.asarray(scores16, dtype=np.float64)
    y = np.asarray(y, dtype=np.int64)
    m = s.max(axis=1)
    lse = np.log(np.exp(s - m[:, None]).sum(axis=1))
    ok = (y >= 0) & (y < s.shape[1])
    sy = s[np.arange(len(s)), np.where(ok, y, 0)]
    return np.where(ok, (sy - m) - lse, np.nan)


def logp_bound(scores16, y):
    """Bound on |V - T| for V the fp32 value the device (or torch) forms before the final fp16 rounding.

    With u = 2^-24, d_k = s_k - m <= 0 and S = sum_k exp(d_k) >= 1 (the maximum contributes exp(0) = 1 exactly):
      - each argument d_k is rounded once: |fl(d_k) - d_k| <= u|d_k|, so exp moves by at most exp(d_k) u |d_k| <= u / e;
        over K columns at most K u / e in S;
      - expf is within 2 ulp (<= 4u relative); the running maximum rescales a partial sum by one more expf and one
        product at most n_pass times in a thread and twice in the four-lane merge (<= 6u relative each, the argument
        term being absorbed as above); fp32 summation of K + n_pass + 2 positive terms adds at most (K + n_pass + 2) u
        relative.  Together |S^ - S| <= S u (K + 6 (n_pass + 2) + 4) + K u, and S >= 1 gives a relative error
        r = u (2K + 6 (n_pass + 2) + 4) (the second-order terms are covered by the 1.01 factor below);
      - logf is within 1 ulp (<= 2u |log S|), and |log S^ - log S| <= 1.01 r;
      - fl(d_y) - fl(log S^) adds u |d_y| and one rounding of the result, u |T| (1 + ...).
    So |V - T| <= u |d_y| + 1.01 r + 2u log S + 1.01 u |T|.  The fp16 result is then within that plus half an fp16 ulp
    of T, and within one fp16 ulp of fp16(T) wherever the fp32 error stays below half an ulp."""
    s = np.asarray(scores16, dtype=np.float64)
    k = s.shape[1]
    n_pass = (k + 95) // 96
    y = np.asarray(y, dtype=np.int64)
    m = s.max(axis=1)
    lse = np.log(np.exp(s - m[:, None]).sum(axis=1))
    ok = (y >= 0) & (y < k)
    dy = s[np.arange(len(s)), np.where(ok, y, 0)] - m
    t = dy - lse
    r = U * (2 * k + 6 * (n_pass + 2) + 4)
    return U * np.abs(dy) + 1.01 * r + 2 * U * lse + 1.01 * U * np.abs(t)


def scene_loss(logp16, y, ignore=IGNORE, k=None):
    """fp64 value and fp16 result of the scene loss from the per-row fp16 logp: mean of -logp over labelled rows."""
    y = np.asarray(y, dtype=np.int64)
    lab = y != ignore
    if k is not None:
        lab &= (y >= 0) & (y < k)
    terms = -np.asarray(logp16, dtype=np.float64)[lab]
    v = terms.sum() / len(terms) if len(terms) else float('nan')
    return v, np.float16(v), terms


def loss_bound(terms, row_bound):
    """Allowed |loss - fp64 mean|: the fp32 sum-order term (rows 2^-24) sum|terms| of torch's accumulation, the mean of the
    per-row allowances (row_bound: each row's distance between its fp16 logp and the reference term), half an fp16 ulp."""
    rows = len(terms)
    if rows == 0:
        return float('nan')
    v = float(np.mean(terms))
    return rows * U * float(np.abs(terms).sum()) + float(np.mean(row_bound)) + 0.5 * float(ulp16(v))


def argmax_nan_first(scores):
    """The first NaN of a row if it holds one, else the first maximum (vote.cuh)."""
    s = np.asarray(scores, dtype=np.float32)
    nan = np.isnan(s)
    has = nan.any(axis=1)
    first_nan = np.argmax(nan, axis=1)
    first_max = np.argmax(np.where(nan, -np.inf, s), axis=1)
    return np.where(has, first_nan, first_max).astype(np.int64)


def intersection_and_union(output, target, K, ignore_index=IGNORE):
    """util/util.py:132-145 (intersectionAndUnionGPU) on the CPU: float32 histc counts (intersection, union, target)."""
    output = torch.as_tensor(output).clone().view(-1)
    target = torch.as_tensor(target).view(-1)
    output[target == ignore_index] = ignore_index
    intersection = output[output == target]
    area_intersection = torch.histc(intersection.float(), bins=K, min=0, max=K - 1)
    area_output = torch.histc(output.float(), bins=K, min=0, max=K - 1)
    area_target = torch.histc(target.float(), bins=K, min=0, max=K - 1)
    area_union = area_output + area_target - area_intersection
    return area_intersection, area_union, area_target


class AverageMeter:
    """util/util.py:86-102."""

    def __init__(self):
        self.val = 0
        self.avg = 0
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def validate_tail(scenes, batch_size=1):
    """run/distill.py:432-446 over per-scene (loss_item, intersection, union, target), the vectors as float32 NumPy arrays
    the way ``.cpu().numpy()`` hands them over."""
    loss_meter, im, um, tm = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
    for loss, inter, union, target in scenes:
        im.update(inter), um.update(union), tm.update(target)
        loss_meter.update(loss, batch_size)
    iou_class = im.sum / (um.sum + 1e-10)
    accuracy_class = im.sum / (tm.sum + 1e-10)
    mIoU = np.mean(iou_class)
    mAcc = np.mean(accuracy_class)
    allAcc = sum(im.sum) / (sum(tm.sum) + 1e-10)
    return loss_meter.avg, mIoU, mAcc, allAcc


def same(a, b):
    """Bit equality of two results of validate_tail, element types included (NaN equal to NaN)."""
    for x, y in zip(a, b):
        if type(x) is not type(y):
            return False
        fx, fy = float(x), float(y)
        if not (fx == fy or (math.isnan(fx) and math.isnan(fy))):
            return False
    return len(a) == len(b)


def device_counts(pred, y, classes, k, ignore=IGNORE):
    """int64 [3, classes] the device counts for one scene, and its bad-label count: rows whose label lies outside [0, K)
    and is not the ignore label are left out; the others follow intersectionAndUnionGPU."""
    pred = np.asarray(pred, dtype=np.int64).copy()
    y = np.asarray(y, dtype=np.int64)
    bad = (y != ignore) & ((y < 0) | (y >= k))
    pred, y = pred[~bad], y[~bad]
    pred[y == ignore] = ignore
    out = np.zeros((3, classes), dtype=np.int64)
    o_in = (pred >= 0) & (pred < classes)
    t_in = (y >= 0) & (y < classes)
    np.add.at(out[0], pred[o_in & (pred == y)], 1)
    np.add.at(out[1], pred[o_in], 1)
    np.add.at(out[2], y[t_in], 1)
    return out, int(bad.sum())
