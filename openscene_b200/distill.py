"""Distillation step and data-parallel plumbing (run/distill.py:121-150, 295-334, 403-447) on the drop-in surface.

One process per GPU, scenes sharded by rank (``DistributedSampler`` semantics, run/distill.py:183-184), plain
per-rank BatchNorm (the reference never enables SyncBN, run/distill.py:108), gradient all-reduce through
``DistributedDataParallel`` over NCCL, three small metric all-reduces in validation (run/distill.py:429-431)."""
import math
import os

import torch
import torch.distributed as dist

from . import _cabi as C


def init_distributed(backend=None):
    """Rendezvous from the torchrun environment; returns (rank, local_rank, world)."""
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    if world > 1 and not dist.is_initialized():
        backend = backend or ('nccl' if torch.cuda.is_available() else 'gloo')
        dist.init_process_group(backend)
    return rank, local, world


def shard_indices(n_items, rank, world, epoch=0, shuffle=True, seed=0):
    """Indices this rank processes: DistributedSampler's rule (pad by wrapping so every rank gets the same count)."""
    if shuffle:
        g = torch.Generator().manual_seed(seed + epoch)
        order = torch.randperm(n_items, generator=g).tolist()
    else:
        order = list(range(n_items))
    per = (n_items + world - 1) // world
    pad = per * world - n_items
    if pad > 0:                                   # DistributedSampler: repeat the list when pad > len (n_items < world / 2)
        order += (order * math.ceil(pad / len(order)))[:pad]
    return order[rank:per * world:world]


def distill_loss(output_3d, feat_3d, loss_type='cosine'):
    """run/distill.py:324-328."""
    feat_3d = feat_3d.to(output_3d.dtype)
    if loss_type == 'cosine':
        return (1 - torch.nn.CosineSimilarity()(output_3d, feat_3d)).mean()
    if loss_type == 'l1':
        return torch.nn.L1Loss()(output_3d, feat_3d)
    raise NotImplementedError


class _PassThrough(torch.nn.Module):
    def forward(self, x):
        return x


def _late_head(model):
    """(network, final) when the network ends in a bias-free 1x1x1 convolution applied row by row
    (``self.final(out).F``, models/mink_unet.py:108-114,174), looked up through DDP (.module) and DisNet (.net3d)."""
    m = model.module if hasattr(model, 'module') else model
    m = m.net3d if hasattr(m, 'net3d') else m
    fin = getattr(m, 'final', None)
    if fin is not None and getattr(fin, 'use_mm', False) and getattr(fin, 'bias', None) is None and fin.kernel.dim() == 2:
        return m, fin
    return None, None


def distill_step(model, optimizer, coords, feats, feat_3d, mask, loss_type='cosine', translate=True, late_head=True):
    """One training step, run/distill.py:311-334: random integer translation of the voxel grid (:315), forward
    (BN in train mode), row select by ``mask`` (:322), cosine / L1 loss, backward (+ DDP all-reduce), Adam step.

    late_head: the last layer is a 1x1x1 convolution, i.e. a per-row linear map, and the loss only sees the ``mask`` rows
    (20 k of ~200 k voxels): ``final(x)[mask] == x[mask] @ W`` exactly, so the 96 -> 768 layer, its two gradients and the
    [N, 768] select / scatter pair run on the supervised rows only.  Same loss, same gradients (up to fp32 summation order)."""
    import MinkowskiEngine as ME
    if translate:
        coords = coords.clone()
        coords[:, 1:4] += (torch.rand(3) * 100).type_as(coords)
    sinput = ME.SparseTensor(feats.cuda(non_blocking=True), coords.cuda(non_blocking=True))
    net, fin = _late_head(model) if late_head else (None, None)
    if net is not None:
        net.final = _PassThrough()                    # the network returns the 96-d rows ...
        try:
            rows = model(sinput)
        finally:
            net.final = fin
        output_3d = rows[mask.to(rows.device)] @ fin.kernel          # ... and the head runs on the supervised rows
    else:
        output_3d = model(sinput)
        output_3d = output_3d[mask.to(output_3d.device)]
    loss = distill_loss(output_3d, feat_3d.to(output_3d.device), loss_type)
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return loss.detach()


def fused_distill_step(engine, optimizer, coords, feats, feat_3d, mask, loss_type='cosine', translate=True):
    """``distill_step`` on the fused engine: the same random translation, loss, zero_grad, backward and optimiser step, with
    the forward and backward of ``engine.forward_train(..., rows=mask)`` (a ``FusedMinkUNet(model, batch_stats=True)``).
    With more than one process, the engine must all-reduce the gradients itself: build it with
    ``process_group=dist.group.WORLD`` (a DistributedDataParallel wrapper's forward, which the engine bypasses, never runs).
    The loss stays per rank, as in run/distill.py."""
    refuse_local_engine(engine, 'fused_distill_step')
    if translate:
        coords = coords.clone()
        coords[:, 1:4] += (torch.rand(3) * 100).type_as(coords)
    dev = engine.device
    out = engine.forward_train(coords.to(dev, non_blocking=True), feats.to(dev, non_blocking=True), rows=mask.to(dev))
    loss = distill_loss(out, feat_3d.to(dev), loss_type)
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return loss.detach()


def fused_cosine_step(engine, optimizer, coords, feats, feat_3d, mask, translate=True):
    """``fused_distill_step`` with the cosine loss on the engine's device head: the same random translation, zero_grad,
    backward and optimiser step, with ``engine.forward_train_cosine`` in place of ``forward_train`` + ``distill_loss``, so
    the [M, C] output rows and their gradient are never materialised.  ``feat_3d`` is cast to fp16 on the engine's device
    (the dtype run/distill.py's targets have).  The L1 loss has its own device head: ``fused_l1_step``."""
    return _fused_head_step(engine, optimizer, coords, feats, feat_3d, mask, translate, 'fused_cosine_step',
                            engine.forward_train_cosine)


def fused_l1_step(engine, optimizer, coords, feats, feat_3d, mask, translate=True):
    """``fused_distill_step(..., loss_type='l1')`` on the engine's device L1 head: ``fused_cosine_step`` with
    ``engine.forward_train_l1`` (the same translation draw, zero_grad, backward and optimiser step; bound ``optim.Adam`` /
    ``optim.SGD``, ``torch.optim`` and ``process_group`` engines alike)."""
    return _fused_head_step(engine, optimizer, coords, feats, feat_3d, mask, translate, 'fused_l1_step',
                            engine.forward_train_l1)


def _fused_head_step(engine, optimizer, coords, feats, feat_3d, mask, translate, what, forward):
    refuse_local_engine(engine, what)
    if translate:
        coords = coords.clone()
        coords[:, 1:4] += (torch.rand(3) * 100).type_as(coords)
    dev = engine.device
    loss = forward(coords.to(dev, non_blocking=True), feats.to(dev, non_blocking=True), feat_3d.to(dev, torch.float16),
                   mask.to(dev))
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return loss.detach()


def refuse_local_engine(engine, what):
    """Refuse a fused engine that keeps its gradients local when more than one process trains."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        pg = engine.process_group
        if pg is None or dist.get_world_size(group=pg) < 2:
            raise RuntimeError(f"{what}: the fused engine all-reduces gradients only when built with a process group "
                               f"(world size {dist.get_world_size()}): FusedMinkUNet(model, batch_stats=True, "
                               f"process_group=dist.group.WORLD)")


def wrap_ddp(model, device=None):
    if dist.is_initialized() and dist.get_world_size() > 1:
        ids = [device.index] if device is not None and device.type == 'cuda' else None
        # gradients live inside the all-reduce buckets (no copy in / out), 16 MB buckets: the first all-reduce starts after the
        # decoder's gradients, the last (exposed) one carries the stem and the first encoder stage only
        return torch.nn.parallel.DistributedDataParallel(model, device_ids=ids, gradient_as_bucket_view=True, bucket_cap_mb=16)
    return model


def allreduce_sum(*tensors):
    """run/distill.py:429-431: in-place SUM of the per-class intersection / union / target vectors."""
    if dist.is_initialized() and dist.get_world_size() > 1:
        for t in tensors:
            dist.all_reduce(t)
    return tensors


class DeviceValidation:
    """The tail of run/distill.py: validate() after the forward (:420-431 per scene, :437-446 at the end) on the device.

    Per scene, ``add`` issues one product of the voxel rows with the text embeddings (``osb_match_ce``) that leaves the
    scene's fp16 cross-entropy loss (``CrossEntropyLoss(ignore_index)`` on ``output[inds_reverse].half() @ text.t()``) and
    its ``intersectionAndUnionGPU`` counts on the device, without a host synchronisation.  ``end`` reads everything once
    and replays the reference's host arithmetic scene by scene (float32 ``AverageMeter`` sums, the ``1e-10`` terms, the
    loss meter in Python floats), so it returns the reference's ``(loss_avg, mIoU, mAcc, allAcc)`` on the same scores.

    With a process group, ``end`` sums the stacked per-scene counts over the ranks in one all-reduce before the replay,
    where the reference all-reduces the three vectors of every scene; every rank must have added the same number of scenes.
    The loss stays per rank, as in the reference.  A label outside ``[0, K)`` other than ``ignore_label`` (a device assert
    in torch) leaves its row out of the loss and the counts and makes ``end`` raise ``IndexError``."""

    def __init__(self, text_features, classes, ignore_label=255, process_group=None):
        C.require_cuda(text_features, 'text_features')
        if text_features.dim() != 2 or text_features.dtype != torch.float16:
            raise ValueError(f"DeviceValidation: text_features must be fp16 [K, C], got {text_features.dtype} "
                             f"{tuple(text_features.shape)}")
        k, c = text_features.shape
        if not 1 <= k <= 480 or c not in (512, 768):
            raise ValueError(f"DeviceValidation: K={k} outside 1..480 or width {c} not 512 / 768")
        if not 1 <= int(classes) <= 512:
            raise ValueError(f"DeviceValidation: classes={classes} outside 1..512")
        self.text = text_features.contiguous()
        self.device = self.text.device
        self.classes = int(classes)
        self.ignore_label = int(ignore_label)
        self.process_group = process_group
        self.begin()

    def begin(self):
        """Start a validation: forget the scenes added so far."""
        self.n = 0
        self._grow(64)
        self._ws = torch.empty(0, dtype=torch.float64, device=self.device)

    def _grow(self, cap):
        """Per-scene storage for ``cap`` scenes: the fp16 loss, the [3, classes] counts and the bad-label count."""
        loss = torch.empty(cap, dtype=torch.float16, device=self.device)
        areas = torch.zeros((cap, 3, self.classes), dtype=torch.int64, device=self.device)
        bad = torch.zeros(cap, dtype=torch.int32, device=self.device)
        if self.n:
            loss[:self.n] = self._loss[:self.n]
            areas[:self.n] = self._areas[:self.n]
            bad[:self.n] = self._bad[:self.n]
        self._loss, self._areas, self._bad = loss, areas, bad

    def add(self, output, inds_reverse, label):
        """One scene: ``output`` the network's [N_vox, C] rows (fp32 or fp16), ``inds_reverse`` the voxel of every point
        (or None: one point per row), ``label`` int32 / int64 per point.  No synchronisation."""
        C.require_cuda(output, 'output')
        if output.dim() != 2 or output.shape[1] != self.text.shape[1]:
            raise ValueError(f"DeviceValidation.add: output {tuple(output.shape)} against text width {self.text.shape[1]}")
        feat = output.detach().contiguous()
        if feat.dtype not in (torch.float16, torch.float32):
            feat = feat.float()
        n_vox = feat.shape[0]
        inv = None
        if inds_reverse is not None:
            inv = inds_reverse.to(device=self.device, dtype=torch.int64, non_blocking=True).contiguous().view(-1)
        n_pts = inv.numel() if inv is not None else n_vox
        lab = torch.as_tensor(label).to(self.device, non_blocking=True).contiguous().view(-1)
        if lab.dtype not in (torch.int32, torch.int64):
            lab = lab.long()
        if lab.numel() != n_pts:
            raise ValueError(f"DeviceValidation.add: {lab.numel()} labels for {n_pts} points")
        if n_vox == 0:
            raise ValueError("DeviceValidation.add: the scene has no voxel rows")
        if self.n == self._loss.numel():
            self._grow(2 * self.n)
        need = 2 * ((n_pts + 127) // 128)
        if self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.float64, device=self.device)
        i = self.n
        with torch.cuda.device(self.device):
            C.call('osb_match_ce', C.ptr(feat), int(feat.dtype == torch.float16), n_vox, feat.shape[1], C.ptr(inv), n_pts,
                   C.ptr(self.text), self.text.shape[0], C.ptr(lab), int(lab.dtype == torch.int64), self.ignore_label,
                   self.classes, None, None, C.c_void_p(self._loss.data_ptr() + 2 * i), C.ptr(self._areas[i]),
                   C.c_void_p(self._bad.data_ptr() + 4 * i), C.ptr(self._ws), 8 * self._ws.numel(), C.stream_ptr())
        self.n += 1

    def end(self, weight=1):
        """``(loss_avg, mIoU, mAcc, allAcc)`` as validate() returns them, ``weight`` the ``args.batch_size`` of its
        ``loss_meter.update``.  One read of the device state (SYNC); with a process group, one all-reduce of the counts."""
        n = self.n
        return validation_result(self._loss[:n], self._areas[:n], self._bad[:n], weight, self.process_group)


def validation_result(losses, areas, bad, weight=1, process_group=None, owner='DeviceValidation'):
    """DeviceValidation.end (and train_mink.DeviceMinkValidation.end, ``owner`` naming it in errors) on its per-scene state
    (any device): ``losses`` fp16 or fp32 [n], ``areas`` int64 [n, 3, classes] (intersection, output, target), ``bad`` int32
    [n] counts of labels outside [0, K) other than the ignore label."""
    import numpy as np
    n = losses.shape[0]
    bad = bad.cpu()
    world = dist.get_world_size(group=process_group) if process_group is not None else 1
    if world > 1:
        on_cpu = dist.get_backend(process_group) == 'gloo'
        st = torch.tensor([n, -n, int(bool(bad.any()))], dtype=torch.int64, device='cpu' if on_cpu else areas.device)
        dist.all_reduce(st, op=dist.ReduceOp.MAX, group=process_group)
        hi, lo, any_bad = int(st[0]), -int(st[1]), int(st[2])
        if hi != lo:
            raise RuntimeError(f"{owner}.end: the ranks added between {lo} and {hi} scenes (this rank {n}); "
                               f"every rank must validate the same number of scenes")
        if any_bad and not bool(bad.any()):
            raise IndexError(f"{owner}.end: another rank saw labels outside [0, K) other than the ignore label")
    hit = torch.nonzero(bad).view(-1)
    if hit.numel():
        s = int(hit[0])
        raise IndexError(f"{owner}.end: scene {s} (0-based, in add() order) has {int(bad[s])} labels outside "
                         f"[0, K) other than the ignore label")
    if world > 1:
        areas = areas.cpu() if on_cpu else areas.clone()
        dist.all_reduce(areas, group=process_group)
    areas = areas.cpu().numpy()
    losses = losses.float().cpu().numpy()
    # run/distill.py:432-441 scene by scene: util.AverageMeter over the float32 vectors (sum += val * 1) and over
    # loss.item() with n = args.batch_size, in Python floats
    loss_sum, loss_count = 0, 0
    inter_sum = union_sum = target_sum = 0
    for s in range(n):
        inter, out, tgt = (areas[s, j].astype(np.float32) for j in range(3))
        inter_sum += inter * 1
        union_sum += (out + tgt - inter) * 1
        target_sum += tgt * 1
        loss_sum += float(losses[s]) * weight
        loss_count += weight
    iou_class = inter_sum / (union_sum + 1e-10)
    accuracy_class = inter_sum / (target_sum + 1e-10)
    mIoU = np.mean(iou_class)
    mAcc = np.mean(accuracy_class)
    allAcc = sum(inter_sum) / (sum(target_sum) + 1e-10)
    return (loss_sum / loss_count if loss_count else 0), mIoU, mAcc, allAcc


def poly_learning_rate(base_lr, curr_iter, max_iter, power=0.9):
    """util/util.py poly schedule used at run/distill.py:341."""
    return base_lr * (1 - float(curr_iter) / max_iter) ** power
