"""NumPy / fp64 restatement of the supervised validation tail of run/train_mink.py (validate(), :366-384) as
``osb_ce_head_eval`` computes it over points, and of train()'s per-step meters (:285-296, :327-331).  The reference is
restated here, not imported."""
import numpy as np

from tests import valce_ref as R

U = R.U
IGNORE = R.IGNORE


def point_head(z_rows, row_of_point, y, ignore=IGNORE):
    """fp64 terms of the point-walking head from the logits of the rows each point reads: ``z_rows`` [n_rows, C],
    ``row_of_point`` [n_pts] (the row every point reads), ``y`` [n_pts].  Returns (loss, pred, counts [3, C], bad): the mean
    of lse - z[y] over points with y in [0, C) (NaN when there is none), the first-NaN / first-maximum argmax, the counts
    of intersectionAndUnionGPU with bad labels left out, and the number of bad labels."""
    z = np.asarray(z_rows, dtype=np.float64)[np.asarray(row_of_point, dtype=np.int64)]
    y = np.asarray(y, dtype=np.int64)
    c = z.shape[1]
    pred = argmax_nan_first64(z)
    counts, bad = R.device_counts(pred, y, c, c, ignore)
    lab = (y != ignore) & (y >= 0) & (y < c)
    if lab.any():
        zl = z[lab]
        m = zl.max(axis=1)
        lse = m + np.log(np.exp(zl - m[:, None]).sum(axis=1))
        loss = float(np.mean(lse - zl[np.arange(len(zl)), y[lab]]))
    else:
        loss = float('nan')
    return loss, pred, counts, bad


def argmax_nan_first64(z):
    z = np.asarray(z, dtype=np.float64)
    nan = np.isnan(z)
    has = nan.any(axis=1)
    return np.where(has, np.argmax(nan, axis=1), np.argmax(np.where(nan, -np.inf, z), axis=1)).astype(np.int64)


def fp32_loss_bound(z_rows, row_of_point, y, ignore=IGNORE):
    """Allowed |loss - fp64 loss| for a loss formed from fp32 logits in fp32 arithmetic: per term lse - z[y], the
    log-sum-exp over C classes (C + 6 roundings of order u (|lse| + 1)) and the difference (u |term|); then the mean, summed in
    fp32 as torch's nll_loss reduces (n u sum|terms| / n), or in fp64 as the device does (covered by the same term)."""
    z = np.asarray(z_rows, dtype=np.float64)[np.asarray(row_of_point, dtype=np.int64)]
    y = np.asarray(y, dtype=np.int64)
    c = z.shape[1]
    lab = (y != ignore) & (y >= 0) & (y < c)
    if not lab.any():
        return float('nan')
    zl = z[lab]
    m = zl.max(axis=1)
    lse = m + np.log(np.exp(zl - m[:, None]).sum(axis=1))
    terms = lse - zl[np.arange(len(zl)), y[lab]]
    row = U * (2 * c + 8) * (np.abs(lse) + np.abs(m) + 1) + U * np.abs(terms)
    n = len(terms)
    return float(n * U * np.abs(terms).sum() / n + row.mean() + U * abs(terms.mean()))


class TrainMeters:
    """train()'s meters, literally: per step the histc vectors as float32 NumPy arrays, loss.item() with args.batch_size."""

    def __init__(self):
        self.loss, self.inter, self.union, self.target = (R.AverageMeter() for _ in range(4))
        self.steps = []

    def step(self, loss_item, inter=None, union=None, target=None, batch_size=1):
        out = {}
        if inter is not None:
            self.inter.update(inter)
            self.union.update(union)
            self.target.update(target)
            accuracy = sum(self.inter.val) / (sum(self.target.val) + 1e-10)
        self.loss.update(loss_item, batch_size)
        out['loss'] = self.loss.val
        if inter is not None:
            out.update(accuracy=accuracy, mIoU=np.mean(inter / (union + 1e-10)), mAcc=np.mean(inter / (target + 1e-10)),
                       allAcc=accuracy)
        self.steps.append(out)
        return out

    def totals(self):
        if self.inter.count == 0:
            return self.loss.avg, None, None, None
        iou_class = self.inter.sum / (self.union.sum + 1e-10)
        accuracy_class = self.inter.sum / (self.target.sum + 1e-10)
        return (self.loss.avg, np.mean(iou_class), np.mean(accuracy_class),
                sum(self.inter.sum) / (sum(self.target.sum) + 1e-10))


def same_steps(a, b):
    """Bit equality of two lists of per-step dicts (types included)."""
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if sorted(x) != sorted(y) or not R.same([x[k] for k in sorted(x)], [y[k] for k in sorted(y)]):
            return False
    return True
