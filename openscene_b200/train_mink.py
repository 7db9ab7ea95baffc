"""Fully supervised training step of the 3D baseline (run/train_mink.py:270-287) on the drop-in surface and on the fused engine.

The step: random integer shift of coordinate columns 0..2 (the reference's ``coords[:, :3]``; with (batch, x, y, z) rows the
batch index moves with x and y, which keeps scenes apart and stays below the coordinate manager's 1024 batch ids), forward
with BatchNorm in train mode, ``CrossEntropyLoss(ignore_index=255)`` over every voxel, zero_grad / backward / optimiser step
(SGD, momentum 0.9, weight decay 1e-4 in config/*/mink.yaml), and ``output.max(1)[1]`` for ``intersectionAndUnionGPU``.

``DeviceMinkValidation`` runs validate()'s per-scene tail on the eval engine and ``DeviceTrainMeter`` keeps train()'s per-step
meters on the device; both read the device once and replay the reference's host arithmetic."""
import torch
import torch.nn.functional as F

from .distill import refuse_local_engine, validation_result


def _translate(coords):
    coords = coords.clone()
    coords[:, :3] += (torch.rand(3) * 100).type_as(coords)
    return coords


def train_step(model, optimizer, coords, feats, labels, ignore_label=255, translate=True):
    """run/train_mink.py:270-287 on the module path.  Returns (loss, pred) with pred = output.max(1)[1] (int64, caller order)."""
    import MinkowskiEngine as ME
    if translate:
        coords = _translate(coords)
    sinput = ME.SparseTensor(feats.cuda(non_blocking=True), coords.cuda(non_blocking=True))
    label = labels.cuda(non_blocking=True)
    output = model(sinput)
    loss = F.cross_entropy(output, label, ignore_index=ignore_label)
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return loss.detach(), output.detach().max(1)[1]


def fused_train_step(engine, optimizer, coords, feats, labels, ignore_label=255, translate=True):
    """``train_step`` on the fused engine (``FusedMinkUNet(model, batch_stats=True)``): the same random shift, loss, zero_grad,
    backward and optimiser step, with ``engine.forward_train_ce``.  Returns (loss, pred) as train_step.
    With more than one process, build the engine with ``process_group=dist.group.WORLD`` (distill.refuse_local_engine); the
    loss and pred stay per rank, as in run/train_mink.py."""
    refuse_local_engine(engine, 'fused_train_step')
    if translate:
        coords = _translate(coords)
    dev = engine.device
    loss, pred = engine.forward_train_ce(coords.to(dev, non_blocking=True), feats.to(dev, non_blocking=True), labels.to(dev),
                                         ignore_index=ignore_label)
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return loss.detach(), pred


class DeviceMinkValidation:
    """run/train_mink.py: validate() (:349-393) on the eval engine: per scene the forward and its tail (the
    ``output[inds_reverse]`` gather, ``CrossEntropyLoss(ignore_index)``, ``output.max(1)[1]`` and ``intersectionAndUnionGPU``)
    in ``engine.forward_eval_ce``, whose final launch leaves the scene's fp32 loss, its ``[3, classes]`` counts and its
    bad-label count on the device.  ``add`` does not synchronise; ``end`` reads everything once and replays the reference's
    host arithmetic (distill.validation_result: float32 ``AverageMeter`` sums, the ``1e-10`` terms, the loss meter in Python
    floats), so it returns validate()'s ``(loss_avg, mIoU, mAcc, allAcc)`` on the same logits.

    ``engine`` is an eval-mode ``FusedMinkUNet(model.eval())`` with a head of ``classes`` outputs.  With a process group,
    ``end`` sums the stacked per-scene counts over the ranks in one all-reduce, where the reference all-reduces the three
    vectors of every scene; every rank must add the same number of scenes, and the loss stays per rank.  A label outside
    ``[0, classes)`` other than ``ignore_label`` (a device assert in torch) leaves its point out of the loss and the counts
    and makes ``end`` raise ``IndexError`` naming the first such scene."""

    def __init__(self, engine, classes, ignore_label=255, process_group=None):
        if engine.batch_stats:
            raise ValueError("DeviceMinkValidation: validate() runs the model in eval mode; pass FusedMinkUNet(model.eval())")
        if int(classes) != engine.out_channels:
            raise ValueError(f"DeviceMinkValidation: classes={classes} but the network has {engine.out_channels} outputs")
        self.engine = engine
        self.device = engine.device
        self.classes = int(classes)
        self.ignore_label = int(ignore_label)
        self.process_group = process_group
        self.begin()

    def begin(self):
        """Start a validation: forget the scenes added so far."""
        self.n = 0
        self._grow(64)

    def _grow(self, cap):
        """Per-scene storage for ``cap`` scenes: the fp32 loss, the [3, classes] counts and the bad-label count."""
        loss = torch.empty(cap, dtype=torch.float32, device=self.device)
        areas = torch.zeros((cap, 3, self.classes), dtype=torch.int64, device=self.device)
        bad = torch.zeros(cap, dtype=torch.int32, device=self.device)
        if self.n:
            loss[:self.n] = self._loss[:self.n]
            areas[:self.n] = self._areas[:self.n]
            bad[:self.n] = self._bad[:self.n]
        self._loss, self._areas, self._bad = loss, areas, bad

    def add(self, coords, feats, inds_reverse, label):
        """One scene as the loader hands it over: ``coords`` int32 [N_vox, 4], ``feats`` [N_vox, 3], ``inds_reverse`` the
        voxel of every point (or None: one point per voxel), ``label`` int32 / int64 per point.  No synchronisation."""
        if self.n == self._loss.numel():
            self._grow(2 * self.n)
        i, dev = self.n, self.device
        self.engine.forward_eval_ce(coords.to(dev, non_blocking=True), feats.to(dev, non_blocking=True), label, inds_reverse,
                                    self._loss[i:i + 1], self._areas[i], self._bad[i:i + 1], ignore_index=self.ignore_label)
        self.n += 1

    def end(self, weight=1):
        """``(loss_avg, mIoU, mAcc, allAcc)`` as validate() returns them, ``weight`` the ``args.batch_size`` of its
        ``loss_meter.update``.  One read of the device state (SYNC); with a process group, one all-reduce of the counts."""
        n = self.n
        return validation_result(self._loss[:n], self._areas[:n], self._bad[:n], weight, self.process_group,
                                 owner='DeviceMinkValidation')


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


class DeviceTrainMeter:
    """The per-step bookkeeping of run/train_mink.py: train() (:285-342), and of run/distill.py: distill() without counts,
    kept on the device between reads.

    ``add(loss, pred, label)`` copies the step's 0-dim loss into a device slot and counts ``pred`` against ``label`` with
    ``osb_intersection_union`` into the step's ``[3, classes]`` slot; it does not synchronise.  ``read(weight)`` reads the
    steps added since the last read at once (one synchronisation) and replays the reference's host arithmetic step by step
    with its NumPy float32 rules: per step ``loss_meter.val``, ``accuracy`` and the ``mIoU / mAcc / allAcc_train_batch``
    scalars, and the running meters (float32 ``AverageMeter`` sums rounded step by step, the loss meter in Python floats).
    ``weight`` is the ``args.batch_size`` of ``loss_meter.update``."""

    def __init__(self, classes, ignore_label=255, device=None):
        if int(classes) < 1:
            raise ValueError(f"DeviceTrainMeter: classes={classes} must be positive")
        self.classes = int(classes)
        self.ignore_label = int(ignore_label)
        self.device = torch.device(device) if device is not None else None
        self.begin()

    def begin(self):
        """Start an epoch: reset the meters and forget the steps not read yet."""
        self.loss_meter, self.intersection_meter = AverageMeter(), AverageMeter()
        self.union_meter, self.target_meter = AverageMeter(), AverageMeter()
        self._counted = []                         # per pending step: whether it has counts
        self._loss = self._areas = None

    def _slots(self, dev):
        i = len(self._counted)
        if self._loss is None or i == self._loss.numel():
            cap = max(64, 2 * i)
            loss = torch.empty(cap, dtype=torch.float32, device=dev)
            areas = torch.empty((cap, 3, self.classes), dtype=torch.int64, device=dev)
            if i:
                loss[:i] = self._loss[:i]
                areas[:i] = self._areas[:i]
            self._loss, self._areas = loss, areas
        return i

    def add(self, loss, pred=None, label=None):
        """One step: ``loss`` the step's 0-dim device loss; ``pred`` (int64, ``output.max(1)[1]``) and ``label`` the step's
        prediction and labels, or both None (distill()).  No synchronisation."""
        from . import _cabi as C
        C.require_cuda(loss, 'loss')
        if (pred is None) != (label is None):
            raise ValueError("DeviceTrainMeter.add: pass both pred and label, or neither")
        if self._counted and (pred is not None) != self._counted[0]:
            raise ValueError("DeviceTrainMeter.add: every step of a read counts pred against label, or none does")
        dev = self.device or loss.device
        i = self._slots(dev)
        self._loss[i].copy_(loss.detach().reshape(()))
        if pred is not None:
            label = label.to(dev, non_blocking=True).reshape(-1)
            pred = pred.to(dev).reshape(-1)
            if pred.numel() != label.numel():
                raise ValueError(f"DeviceTrainMeter.add: {pred.numel()} predictions for {label.numel()} labels")
            if pred.dtype != torch.int64:
                pred = pred.long()
            if label.dtype != torch.int64:
                label = label.long()
            areas = self._areas[i]
            areas.zero_()
            with torch.cuda.device(dev):
                C.call('osb_intersection_union', C.ptr(pred.contiguous()), C.ptr(label.contiguous()), 1, pred.numel(),
                       self.classes, self.ignore_label, C.ptr(areas), C.stream_ptr())
        self._counted.append(pred is not None)

    def read(self, weight=1):
        """(steps, totals): per step added since the last read a dict with ``loss`` (``loss_meter.val``) and, for steps with
        counts, ``accuracy``, ``mIoU``, ``mAcc`` and ``allAcc`` (the ``*_train_batch`` scalars; allAcc is the step's
        accuracy); ``totals`` = train()'s return ``(loss_meter.avg, mIoU, mAcc, allAcc)`` over the epoch so far (the
        metric terms None without counts).  One synchronisation."""
        import numpy as np
        n = len(self._counted)
        steps = []
        if n:
            loss_h = self._loss[:n].to('cpu', non_blocking=True)
            areas_h = self._areas[:n].to('cpu', non_blocking=True) if self._counted[0] else None
            if self._loss.is_cuda:
                torch.cuda.current_stream(self._loss.device).synchronize()
            loss_h = loss_h.numpy()
            areas_h = areas_h.numpy() if areas_h is not None else None
            for s in range(n):
                self.loss_meter.update(float(loss_h[s]), weight)
                step = {'loss': self.loss_meter.val}
                if areas_h is not None:
                    # run/train_mink.py:289-296 and :327-331 on the float32 vectors .cpu().numpy() hands over
                    intersection, area_output, target = (areas_h[s, j].astype(np.float32) for j in range(3))
                    union = area_output + target - intersection
                    self.intersection_meter.update(intersection)
                    self.union_meter.update(union)
                    self.target_meter.update(target)
                    accuracy = sum(self.intersection_meter.val) / (sum(self.target_meter.val) + 1e-10)
                    step.update(accuracy=accuracy, mIoU=np.mean(intersection / (union + 1e-10)),
                                mAcc=np.mean(intersection / (target + 1e-10)), allAcc=accuracy)
                steps.append(step)
            self._counted = []
        return steps, self.totals()

    def totals(self):
        """train()'s ``(loss_meter.avg, mIoU, mAcc, allAcc)`` over the steps read so far (metrics None without counts)."""
        import numpy as np
        if self.intersection_meter.count == 0:
            return self.loss_meter.avg, None, None, None
        im, um, tm = self.intersection_meter, self.union_meter, self.target_meter
        iou_class = im.sum / (um.sum + 1e-10)
        accuracy_class = im.sum / (tm.sum + 1e-10)
        return self.loss_meter.avg, np.mean(iou_class), np.mean(accuracy_class), sum(im.sum) / (sum(tm.sum) + 1e-10)
