"""Fully supervised training step of the 3D baseline (run/train_mink.py:270-287) on the drop-in surface and on the fused engine.

The step: random integer shift of coordinate columns 0..2 (the reference's ``coords[:, :3]``; with (batch, x, y, z) rows the
batch index moves with x and y, which keeps scenes apart and stays below the coordinate manager's 1024 batch ids), forward
with BatchNorm in train mode, ``CrossEntropyLoss(ignore_index=255)`` over every voxel, zero_grad / backward / optimiser step
(SGD, momentum 0.9, weight decay 1e-4 in config/*/mink.yaml), and ``output.max(1)[1]`` for ``intersectionAndUnionGPU``."""
import torch
import torch.nn.functional as F

from .distill import refuse_local_engine


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
