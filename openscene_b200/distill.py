"""Distillation step and data-parallel plumbing (run/distill.py:121-150, 295-334, 403-447) on the drop-in surface.

One process per GPU, scenes sharded by rank (``DistributedSampler`` semantics, run/distill.py:183-184), plain
per-rank BatchNorm (the reference never enables SyncBN, run/distill.py:108), gradient all-reduce through
``DistributedDataParallel`` over NCCL, three small metric all-reduces in validation (run/distill.py:429-431)."""
import math
import os

import torch
import torch.distributed as dist


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


def poly_learning_rate(base_lr, curr_iter, max_iter, power=0.9):
    """util/util.py poly schedule used at run/distill.py:341."""
    return base_lr * (1 - float(curr_iter) / max_iter) ** power
