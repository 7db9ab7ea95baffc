"""Data-parallel training on the fused engine (``FusedMinkUNet(model, batch_stats=True, process_group=pg)``), world size 2:
once over gloo with both ranks on cuda:0 (gloo stages CUDA tensors through the host: correctness only), once over NCCL on
cuda:0 / cuda:1.

Every rank trains on its own scene.  The reference is a single-process replay on one bare engine: from the same parameters it
computes each rank's local gradient (in batch-statistics mode the gradient does not depend on the running buffers), forms
g0 / 2 + g1 / 2 and applies the same optimiser.  Halving and a two-term sum are exact and the engine's backward is
bit-reproducible, so gradients, parameters and running buffers are compared with torch.equal.  Against the
DistributedDataParallel module path the yardstick of tests/test_gpu_engine_train.py applies (ReLU masks flip under the
split-bf16 rounding)."""
import copy
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ARCH, CLASSES = 'MinkUNet18A', 20


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _bufs(model):
    return [b for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)
            for b in (m.running_mean, m.running_var, m.num_batches_tracked)]


def _flat(ts):
    return torch.cat([t.detach().reshape(-1).double() for t in ts])


def _gathered(x):
    """[rank 0's x, rank 1's x]"""
    out = [torch.empty_like(x) for _ in range(dist.get_world_size())]
    dist.all_gather(out, x)
    return out


def _data(r, dev):
    """rank r's scene: config1_50k, seed r; distillation rows and targets, and per-voxel labels (255 ignored)"""
    from openscene_b200 import synth
    from tests.test_gpu_engine_train_ce import _labels
    c = torch.from_numpy(synth.scene('config1_50k', seed=r))
    g = torch.Generator().manual_seed(40 + r)
    f = torch.rand(len(c), 3, generator=g)
    mask = torch.rand(len(c), generator=g) < 0.2
    tgt = torch.randn(int(mask.sum()), 768, generator=g).half()
    return dict(c=c.to(dev), f=f.to(dev), mask=mask.to(dev), tgt=tgt.to(dev), lab=_labels(c, CLASSES).to(dev))


def _model(out, seed, dev):
    from openscene_b200 import synth
    return synth.randomize_bn_stats(synth.build_model(ARCH, out, seed=seed), seed=seed + 100).to(dev).train()


def _construction(rank, dev):
    from openscene_b200 import engine, synth
    m = _model(768, seed=10 + rank, dev=dev)
    engine.FusedMinkUNet(m, batch_stats=True, process_group=dist.group.WORLD)
    ref = _model(768, seed=10, dev=dev)
    for (k, a), b in zip(m.state_dict().items(), ref.state_dict().values()):
        assert torch.equal(a, b), k
    arch = 'MinkUNet18A' if rank == 0 else 'MinkUNet34C'
    with pytest.raises(RuntimeError, match='differ from rank 0'):
        engine.FusedMinkUNet(synth.build_model(arch, 768, seed=0).to(dev).train(), batch_stats=True,
                             process_group=dist.group.WORLD)


def _steps(rank, dev, ce):
    """3 optimiser steps of fused_train_step (ce) or fused_distill_step against the single-process replay on rank 0"""
    from openscene_b200 import distill, engine, train_mink
    data = [_data(r, dev) for r in range(2)]
    out = CLASSES if ce else 768
    model = _model(out, seed=3 + rank, dev=dev)                  # rank 1's own weights are replaced by rank 0's
    eng = engine.FusedMinkUNet(model, batch_stats=True, process_group=dist.group.WORLD)

    def optim(params):
        return (torch.optim.SGD(params, lr=0.01, momentum=0.9, weight_decay=1e-4) if ce
                else torch.optim.Adam(params, lr=1e-3))
    opt = optim(model.parameters())
    if rank == 0:
        rmodel = _model(out, seed=3, dev=dev)
        reng, ropt = engine.FusedMinkUNet(rmodel, batch_stats=True), optim(rmodel.parameters())
    d = data[rank]
    for step in range(3):
        if ce:
            train_mink.fused_train_step(eng, opt, d['c'], d['f'], d['lab'], translate=False)
        else:
            distill.fused_distill_step(eng, opt, d['c'], d['f'], d['tgt'], d['mask'], translate=False)
        gs = _gathered(_flat(p.grad for p in model.parameters()))
        ps = _gathered(_flat(model.parameters()))
        bs = _gathered(_flat(_bufs(model)))
        if rank != 0:
            continue
        start = [b.clone() for b in _bufs(rmodel)]             # rank 0's buffers before this step's forward
        local, after = [], []
        for r in range(2):
            with torch.no_grad():
                for b, s in zip(_bufs(rmodel), start):
                    b.copy_(s)
            rmodel.zero_grad(set_to_none=True)
            dr = data[r]
            if ce:
                loss, _ = reng.forward_train_ce(dr['c'], dr['f'], dr['lab'], ignore_index=255)
            else:
                loss = distill.distill_loss(reng.forward_train(dr['c'], dr['f'], rows=dr['mask']), dr['tgt'])
            loss.backward()
            local.append([p.grad.clone() for p in rmodel.parameters()])
            after.append(_flat(_bufs(rmodel)))
        for p, g0, g1 in zip(rmodel.parameters(), *local):
            p.grad = g0 / 2 + g1 / 2
        ropt.step()
        with torch.no_grad():
            for b, s in zip(_bufs(rmodel), after[0].split([b.numel() for b in _bufs(rmodel)])):
                b.copy_(s.view_as(b).to(b.dtype))
        tag = f"{'fused_train_step' if ce else 'fused_distill_step'} step {step}"
        g = _flat(p.grad for p in rmodel.parameters())
        assert torch.equal(gs[0], gs[1]) and torch.equal(gs[0], g), f"{tag}: gradients"
        assert torch.equal(ps[0], ps[1]) and torch.equal(ps[0], _flat(rmodel.parameters())), f"{tag}: parameters"
        # each rank's buffers moved from rank 0's: both forwards started from the broadcast buffers
        assert torch.equal(bs[0], after[0]) and torch.equal(bs[1], after[1]), f"{tag}: running buffers"


def _against_ddp(rank, dev):
    """one step of the fused data-parallel step and of the DistributedDataParallel module path from the same state"""
    from openscene_b200 import distill, engine
    from tests.test_gpu_engine_train import _Keep, _grads_close, _perturbed
    d = _data(rank, dev)
    base = _model(768, seed=5, dev=dev)
    m_ddp = distill.wrap_ddp(copy.deepcopy(base), device=dev)
    m_pt = distill.wrap_ddp(_perturbed(copy.deepcopy(base)), device=dev)
    m_eng = copy.deepcopy(base)
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True, process_group=dist.group.WORLD)
    torch.manual_seed(0)
    l_ddp = float(distill.distill_step(m_ddp, _Keep(m_ddp.parameters(), lr=0.0), d['c'], d['f'], d['tgt'], d['mask'],
                                       translate=False))
    distill.distill_step(m_pt, _Keep(m_pt.parameters(), lr=0.0), d['c'], d['f'], d['tgt'], d['mask'], translate=False)
    l_eng = float(distill.fused_distill_step(eng, _Keep(m_eng.parameters(), lr=0.0), d['c'], d['f'], d['tgt'], d['mask'],
                                             translate=False))
    print('rank', rank, 'loss DDP', l_ddp, 'fused', l_eng)
    assert abs(l_ddp - l_eng) <= 1e-4 * abs(l_ddp)
    print('rank', rank, 'worst grad error / (perturbation + 1e-4 max)', _grads_close(m_eng, m_ddp.module, m_pt.module))


def _size_one_group(rank, dev):
    """a group of one rank: the engine's gradients are the bare engine's; a bare engine under world size 2 is refused"""
    from openscene_b200 import distill, engine, train_mink
    own = [dist.new_group([r]) for r in range(dist.get_world_size())][rank]
    d = _data(rank, dev)
    base = _model(768, seed=6, dev=dev)
    m_a, m_b = copy.deepcopy(base), copy.deepcopy(base)
    e_a = engine.FusedMinkUNet(m_a, batch_stats=True, process_group=own)
    e_b = engine.FusedMinkUNet(m_b, batch_stats=True)
    for e in (e_a, e_b):
        distill.distill_loss(e.forward_train(d['c'], d['f'], rows=d['mask']), d['tgt']).backward()
    for (k, a), b in zip(m_a.named_parameters(), m_b.parameters()):
        assert torch.equal(a.grad, b.grad), k
    assert torch.equal(_flat(_bufs(m_a)), _flat(_bufs(m_b)))
    opt = torch.optim.SGD(m_b.parameters(), lr=0.0)
    with pytest.raises(RuntimeError, match='process_group'):
        distill.fused_distill_step(e_b, opt, d['c'], d['f'], d['tgt'], d['mask'])
    with pytest.raises(RuntimeError, match='process_group'):
        train_mink.fused_train_step(e_b, opt, d['c'], d['f'], d['lab'])


def _worker(rank, world, backend, port, devices):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device(devices[rank])
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(minutes=3))
    try:
        _construction(rank, dev)
        _steps(rank, dev, ce=False)
        _steps(rank, dev, ce=True)
        _against_ddp(rank, dev)
        _size_one_group(rank, dev)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _spawn(backend, devices):
    mp.spawn(_worker, args=(2, backend, _free_port(), devices), nprocs=2, join=True)


def test_gloo_two_ranks_on_one_device():
    _spawn('gloo', ['cuda:0', 'cuda:0'])


def test_nccl_two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip(f"NCCL needs one device per rank: {torch.cuda.device_count()} visible")
    _spawn('nccl', ['cuda:0', 'cuda:1'])
