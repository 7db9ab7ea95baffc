"""``FusedMinkUNet.forward_train_l1`` / ``distill.fused_l1_step`` (run/distill.py's L1 step on the device head) against
``distill_loss(forward_train(...), 'l1')`` on the same engine, the module path and torch.optim (the kernels themselves:
tests/test_gpu_l1_head.py).

Against forward_train the trunk forward is the same launch sequence on the same state, so only the head's arithmetic differs
(fp32 W against its split-bf16 pack, the loss in fp64 against torch's fp32 chain).  The loss must agree to 1e-5 relative.  The
gradient of |f - t| jumps where f - t changes sign, so the two arms may disagree on the sign of an element, but only where
|f - t| lies within their difference in f (bounded by the torch arm's measured distance from fp64 plus the device head's
forward bound); fed the device head's signs, the torch arm's backward must give every gradient to
1e-4 of that parameter's largest gradient.  Against the module path the perturbed-module yardstick of
tests/test_gpu_engine_train.py applies, for the reason given there."""
import copy
import datetime
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from openscene_b200 import synth
from tests import replay_ref as R
from tests.test_gpu_engine_train import _Keep, _buffers_close, _grads_close, _perturbed

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


class _Raw:
    """a device byte range as a tensor (the engine's saved activations)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (ptr, False), 'version': 3}


def _scenes(k, width=768, seed=8):
    coords = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=s, batch_index=s)) for s in range(k)])
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(2))
    g = torch.Generator().manual_seed(seed)
    mask = torch.rand(len(coords), generator=g) < 0.2
    tgt = torch.randn(int(mask.sum()), width, generator=g).half()
    return coords.to(DEV), feats.to(DEV), mask.to(DEV), tgt.to(DEV)


def _model(arch, width=768, seed=3):
    return synth.randomize_bn_stats(synth.build_model(arch, width, seed=seed), seed=7).train().to(DEV)


@pytest.mark.parametrize('arch,width', [('MinkUNet18A', 768), ('MinkUNet34C', 768), ('MinkUNet18A', 512),
                                        ('MinkUNet34C', 512)])
def test_matches_forward_train_and_distill_loss(arch, width):
    from openscene_b200 import distill, engine
    from tests import l1_ref
    c, f, mask, tgt = _scenes(1, width)
    model = _model(arch, width)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    loss = eng.forward_train_l1(c, f, tgt, mask)                   # the gradient does not depend on the running buffers
    assert loss.dim() == 0 and loss.dtype == torch.float32
    signs = loss.grad_fn.graph.tape[-1][1][2]
    loss.backward()
    got = [p.grad.clone() for p in model.parameters()]
    model.zero_grad(set_to_none=True)
    out = eng.forward_train(c, f, rows=mask)
    loss_ref = distill.distill_loss(out, tgt, 'l1')
    print(arch, width, 'loss', float(loss.detach()), float(loss_ref.detach()))
    assert abs(float(loss.detach()) - float(loss_ref.detach())) <= 1e-5 * abs(float(loss_ref.detach()))
    # sign disagreements only where |f - t| is within the arms' difference in f: a flip needs |f_torch - t| <=
    # |f_torch - f_device| <= |f_torch - f64| + the device head's forward bound (l1_ref), with f64 = x W on the trunk output
    # both heads read (the split rows decoded) and the fp32 weights
    S = l1_ref.decode(signs, width).to(DEV)
    f_t = out.detach()
    d = f_t - tgt.float()
    flip = S != l1_ref.sgn(d)
    (src, cin, n0), = out.grad_fn.graph.tape[-1][1].srcs
    sel = out.grad_fn.graph.keep[1].long()
    X = R.split_decode(torch.as_tensor(_Raw(src, n0 * 4 * cin), device=DEV).view(n0, -1), cin)[sel]
    Wd = model.final.kernel.detach().double().view(cin, width)
    f64 = X @ Wd
    dev_bound = l1_ref.SLACK * (l1_ref.gam(cin) * (X.abs() @ Wd.abs()) + l1_ref.U * (f64 - tgt.double()).abs())
    near = d.abs().double() <= (f_t.double() - f64).abs() + dev_bound
    print(arch, width, 'sign disagreements', int(flip.sum()), 'of', flip.numel(), 'elements within the arms\' difference',
          int(near.sum()))
    assert not bool((flip & ~near).any())
    # the torch arm's backward fed the device signs: only the head's arithmetic differs
    s = l1_ref.scale(1.0, d.shape[0], width)
    out.backward(s * S.float())
    worst = 0.0
    for (name, p), g in zip(model.named_parameters(), got):
        e, m = float((p.grad - g).abs().max()), float(p.grad.abs().max())
        worst = max(worst, e / (m + 1e-30))
        assert e <= 1e-4 * m, (name, e, m)
    print(arch, width, 'worst gradient difference / largest gradient', worst)


def test_batch_of_four_against_module_path():
    from openscene_b200 import distill, engine
    c, f, mask, tgt = _scenes(4)
    model = _model('MinkUNet18A').cpu()
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    m_pt = _perturbed(copy.deepcopy(model).to(DEV))
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    o_mod, o_eng, o_pt = (_Keep(m.parameters(), lr=0.0) for m in (m_mod, m_eng, m_pt))
    for step in range(2):
        torch.manual_seed(step)
        l_mod = float(distill.distill_step(m_mod, o_mod, c, f, tgt, mask, loss_type='l1'))
        torch.manual_seed(step)
        l_eng = float(distill.fused_l1_step(eng, o_eng, c, f, tgt, mask))
        torch.manual_seed(step)
        distill.distill_step(m_pt, o_pt, c, f, tgt, mask, loss_type='l1')
        print('step', step, 'loss', l_mod, l_eng)
        assert abs(l_mod - l_eng) <= 1e-4 * abs(l_mod)
        print('worst grad error / (perturbation + 1e-4 max)', _grads_close(m_eng, m_mod, m_pt))
        _buffers_close(m_eng, m_mod)


def test_two_identical_steps_are_bit_identical():
    from openscene_b200 import engine
    c, f, mask, tgt = _scenes(1, width=512)
    model = _model('MinkUNet34C', 512)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    out = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        loss = eng.forward_train_l1(c, f, tgt, mask)
        loss.backward()
        out.append((loss.detach().clone(), [p.grad.clone() for p in model.parameters()]))
    assert torch.equal(out[0][0], out[1][0])
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1]))


def _adam_run(model, make_opt, bind, steps=5):
    from openscene_b200 import distill, engine
    c, f, mask, tgt = _scenes(1)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = make_opt(model.parameters())
    if bind:
        opt.bind(eng)
    losses, grads, heads = [], [], []
    for s in range(steps):
        torch.manual_seed(s)
        losses.append(float(distill.fused_l1_step(eng, opt, c, f, tgt, mask)))
        grads.append([p.grad.detach().clone() for p in model.parameters()])
        heads.append(model.final.kernel.detach().clone())
    return losses, grads, heads, [p.detach().clone() for p in model.parameters()]


def test_bound_adam_steps_match_torch_optim():
    """the device Adam bound to the engine (in-place re-pack) against torch.optim.Adam (refresh()): five steps"""
    from openscene_b200 import optim
    base = _model('MinkUNet18A').cpu()
    l_o, g_o, h_o, last_o = _adam_run(copy.deepcopy(base).to(DEV), lambda ps: optim.Adam(ps, lr=1e-3), True)
    l_t, g_t, _, _ = _adam_run(copy.deepcopy(base).to(DEV), lambda ps: torch.optim.Adam(ps, lr=1e-3), False)
    l_o2, _, _, last_o2 = _adam_run(copy.deepcopy(base).to(DEV), lambda ps: optim.Adam(ps, lr=1e-3), True)
    print('losses ours', l_o, 'torch', l_t)
    assert all(torch.equal(a, b) for a, b in zip(g_o[0], g_t[0])), "step 1 starts from the same gradients"
    for a, b in zip(l_o, l_t):
        assert abs(a - b) <= 1e-4 * abs(b)
    assert l_o == l_o2 and all(torch.equal(a, b) for a, b in zip(last_o, last_o2)), "two runs differ"
    # every step reads the head the previous step wrote: the head moves and the loss follows it
    assert not torch.equal(h_o[0], h_o[1]) and l_o[-1] < l_o[0]


def test_steps_reduce_loss_and_eval_engine_refolds():
    from openscene_b200 import distill, engine
    from tests.util import rel_row_err
    c = torch.from_numpy(synth.random_cloud(1200, 18, seed=9))
    f = torch.ones(len(c), 3)
    g = torch.Generator().manual_seed(3)
    mask = torch.rand(len(c), generator=g) < 0.6
    tgt = torch.randn(int(mask.sum()), 512, generator=g).half()
    model = synth.build_model('MinkUNet14A', 512, seed=1).to(DEV).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    model.eval()
    eng_eval = engine.FusedMinkUNet(model)
    out0 = eng_eval(c.to(DEV), f.to(DEV)).clone()
    model.train()
    losses = [float(distill.fused_l1_step(eng, opt, c, f, tgt, mask)) for _ in range(6)]
    assert losses[-1] < losses[0], losses
    model.eval()
    out1 = eng_eval(c.to(DEV), f.to(DEV))
    ref = synth.build_model('MinkUNet14A', 512, seed=1)
    ref.load_state_dict(model.state_dict())
    import MinkowskiEngine as ME
    with torch.no_grad():
        r = ref.to(DEV).eval()(ME.SparseTensor(f.to(DEV), c.to(DEV)))
    assert rel_row_err(out1.cpu().numpy(), r.cpu().numpy()) < 1e-3
    assert rel_row_err(out1.cpu().numpy(), out0.cpu().numpy()) > 1e-3


def test_refusals():
    from openscene_b200 import engine
    c, f, mask, tgt = _scenes(1)
    model = _model('MinkUNet14A')
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    torch.cuda.synchronize()
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(ValueError, match='is on'):
        eng.forward_train_l1(c, f, tgt.cpu(), mask)
    with pytest.raises(TypeError, match='fp16'):
        eng.forward_train_l1(c, f, tgt.float(), mask)
    with pytest.raises(ValueError, match='rows for'):
        eng.forward_train_l1(c, f, tgt[:-1], mask)
    with pytest.raises(ValueError, match='repeated'):
        eng.forward_train_l1(c, f, tgt[:2], torch.tensor([4, 4], device=DEV))
    with pytest.raises(NotImplementedError, match='input features'):
        eng.forward_train_l1(c, f.clone().requires_grad_(), tgt, mask)
    model.eval()
    with pytest.raises(RuntimeError, match='train'):
        eng.forward_train_l1(c, f, tgt, mask)
    model.train()
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())


# ------------------------------------------------------------------------------------------------ two ranks over gloo
def _dp_steps(rank, dev):
    """3 Adam steps of fused_l1_step on two ranks against a single-process replay of the new path on rank 0"""
    from openscene_b200 import distill, engine
    from tests.test_gpu_engine_dp import _bufs, _data, _flat, _gathered
    from tests.test_gpu_engine_dp import _model as dp_model
    data = [_data(r, dev) for r in range(2)]
    model = dp_model(768, seed=3 + rank, dev=dev)                  # rank 1's own weights are replaced by rank 0's
    eng = engine.FusedMinkUNet(model, batch_stats=True, process_group=dist.group.WORLD)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    if rank == 0:
        rmodel = dp_model(768, seed=3, dev=dev)
        reng, ropt = engine.FusedMinkUNet(rmodel, batch_stats=True), torch.optim.Adam(rmodel.parameters(), lr=1e-3)
    d = data[rank]
    for step in range(3):
        distill.fused_l1_step(eng, opt, d['c'], d['f'], d['tgt'], d['mask'], translate=False)
        gs = _gathered(_flat(p.grad for p in model.parameters()))
        ps = _gathered(_flat(model.parameters()))
        bs = _gathered(_flat(_bufs(model)))
        if rank != 0:
            continue
        start = [b.clone() for b in _bufs(rmodel)]
        local, after = [], []
        for r in range(2):
            with torch.no_grad():
                for b, s in zip(_bufs(rmodel), start):
                    b.copy_(s)
            rmodel.zero_grad(set_to_none=True)
            dr = data[r]
            reng.forward_train_l1(dr['c'], dr['f'], dr['tgt'], dr['mask']).backward()
            local.append([p.grad.clone() for p in rmodel.parameters()])
            after.append(_flat(_bufs(rmodel)))
        for p, g0, g1 in zip(rmodel.parameters(), *local):
            p.grad = g0 / 2 + g1 / 2
        ropt.step()
        with torch.no_grad():
            for b, s in zip(_bufs(rmodel), after[0].split([b.numel() for b in _bufs(rmodel)])):
                b.copy_(s.view_as(b).to(b.dtype))
        g = _flat(p.grad for p in rmodel.parameters())
        assert torch.equal(gs[0], gs[1]) and torch.equal(gs[0], g), f"step {step}: gradients"
        assert torch.equal(ps[0], ps[1]) and torch.equal(ps[0], _flat(rmodel.parameters())), f"step {step}: parameters"
        assert torch.equal(bs[0], after[0]) and torch.equal(bs[1], after[1]), f"step {step}: running buffers"


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device(DEV)
    torch.cuda.set_device(dev)
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(minutes=3))
    try:
        _dp_steps(rank, dev)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_gloo_two_ranks_on_one_device():
    from tests.test_gpu_engine_dp import _free_port
    mp.spawn(_worker, args=(2, _free_port()), nprocs=2, join=True)
