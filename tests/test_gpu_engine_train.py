"""``FusedMinkUNet.forward_train`` and its device backward against the fp64 oracle and the module path (the BatchNorm backward
kernels themselves: tests/test_gpu_bn_backward.py).

Gradients through ReLU are discontinuous: an element whose pre-activation lies within the forward's rounding of zero takes the
other branch in one arm, and its whole upstream gradient moves from one BatchNorm sum to the other.  The engine keeps
activations in split-bf16 rows (2^-17) where the module path keeps fp32, so a few dozen of ~6 M elements per layer flip, and
every gradient below that layer moves by about |g| per flip -- up to 1e-2 of the largest gradient, far above 2e-3.  The
yardstick for gradients is therefore the one of tests/test_gpu_unet.py: the module path itself with every convolution kernel
perturbed by 2^-16 relative noise (the operand precision of the split-bf16 path) flips masks the same way, and the engine must
stay within a small multiple of that change (+ 2e-3 of the largest magnitude).  Loss and running buffers are continuous and
keep their direct bounds."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from openscene_b200 import _cabi as C
from openscene_b200 import synth
from tests.util import rel_row_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _to_split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _joined(rows, c):
    out = torch.empty((rows.shape[0], c), dtype=torch.float32, device=DEV)
    C.call('osb_split_to_f32', C.ptr(rows), rows.shape[0], c, C.ptr(out), C.stream_ptr())
    return out


# ---------------------------------------------------------------------------------------------------------------------------
def _perturbed(model, seed=5):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n_, p_ in model.named_parameters():
            if n_.endswith('kernel'):
                p_.mul_(1 + 2.0 ** -16 * torch.randn(p_.shape, generator=g).to(p_.device))
    return model


def _scene(name):
    c = synth.scene(name)
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(2))
    return torch.from_numpy(c).to(DEV), f.to(DEV)


def _bns(model):
    return [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)]


def _buffers_close(a, b, tol=1e-3):
    for x, y in zip(_bns(a), _bns(b)):
        for name in ('running_mean', 'running_var'):
            p, q = getattr(x, name), getattr(y, name)
            assert float((p - q).abs().max()) <= tol * float(q.abs().max()), name
        assert int(x.num_batches_tracked) == int(y.num_batches_tracked)


def _grads_close(ma, mb, mp, tol=2e-3, k=10):
    """ma (engine) against mb (module path), with mp (module path, perturbed kernels) as the yardstick"""
    worst = 0.0
    for (key, a), (_, b), (_, p) in zip(ma.named_parameters(), mb.named_parameters(), mp.named_parameters()):
        e = float((a.grad - b.grad).abs().max())
        e_p = float((p.grad - b.grad).abs().max())
        s = float(b.grad.abs().max())
        worst = max(worst, e / (e_p + 1e-4 * s + 1e-30))
        assert e <= k * e_p + tol * s + 1e-8, (key, e, e_p, s)
    return worst


class _Keep(torch.optim.SGD):            # leaves the weights alone: gradients and buffers stay comparable step after step
    def step(self, closure=None):
        return None


@pytest.mark.parametrize('arch', ['MinkUNet18A', 'MinkUNet34C'])
def test_engine_step_matches_module_path(arch):
    import MinkowskiEngine as ME
    from openscene_b200 import distill, engine
    c, f = _scene('config1_50k')
    g = torch.Generator().manual_seed(8)
    mask = (torch.rand(len(c), generator=g) < 0.2).to(DEV)
    tgt = torch.randn(int(mask.sum()), 768, generator=g).half().to(DEV)
    model = synth.randomize_bn_stats(synth.build_model(arch, 768, seed=3), seed=7).train()
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    m_pt = _perturbed(copy.deepcopy(model).to(DEV))
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    o_mod, o_eng, o_pt = (_Keep(m.parameters(), lr=0.0) for m in (m_mod, m_eng, m_pt))
    for step in range(3):
        torch.manual_seed(step)
        l_mod = float(distill.distill_step(m_mod, o_mod, c, f, tgt, mask, translate=True))
        torch.manual_seed(step)
        l_eng = float(distill.fused_distill_step(eng, o_eng, c, f, tgt, mask, translate=True))
        torch.manual_seed(step)
        distill.distill_step(m_pt, o_pt, c, f, tgt, mask, translate=True)
        print(arch, 'step', step, 'loss', l_mod, l_eng)
        assert abs(l_mod - l_eng) <= 1e-4 * abs(l_mod)
        print('worst grad error / (perturbation + 1e-4 max)', _grads_close(m_eng, m_mod, m_pt))
        _buffers_close(m_eng, m_mod)
    # three Adam steps from the same weights: the two arms stay together
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    o_mod, o_eng = torch.optim.Adam(m_mod.parameters(), lr=1e-3), torch.optim.Adam(m_eng.parameters(), lr=1e-3)
    for step in range(4):
        l_mod = float(distill.distill_step(m_mod, o_mod, c, f, tgt, mask, translate=False))
        l_eng = float(distill.fused_distill_step(eng, o_eng, c, f, tgt, mask, translate=False))
    print(arch, 'after 3 Adam steps', l_mod, l_eng)
    assert abs(l_mod - l_eng) <= 1e-3 * abs(l_mod)


def test_rows_none_matches_model_with_random_upstream_gradient():
    import MinkowskiEngine as ME
    from openscene_b200 import engine
    c, f = _scene('config1_50k')
    model = synth.build_model('MinkUNet18A', 96, seed=4).train()
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    m_pt = _perturbed(copy.deepcopy(model).to(DEV))
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    ref = m_mod(ME.SparseTensor(f, c))
    m_pt(ME.SparseTensor(f, c)).backward(torch.randn(ref.shape, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV))
    out = eng.forward_train(c, f)
    assert out.shape == ref.shape and out.grad_fn is not None
    assert rel_row_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-3
    up = torch.randn(ref.shape, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    ref.backward(up)
    out.backward(up)
    print('worst grad error / (perturbation + 1e-4 max)', _grads_close(m_eng, m_mod, m_pt))
    _buffers_close(m_eng, m_mod)


def test_against_fp64_oracle():
    """the yardstick of tests/test_gpu_unet.py: within a small multiple of what a 2^-16 perturbation of the kernels changes"""
    from openscene_b200 import engine
    from oracle import matching as omatch
    from oracle import me_cpu
    c = synth.scene('tiny')
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(0))
    tgt = torch.randn(len(c), 64, generator=torch.Generator().manual_seed(1))
    m64 = synth.build_model('MinkUNet14A', 64, seed=0, ME=me_cpu.as_module()).double().train()
    mpt = copy.deepcopy(m64)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n_, p_ in mpt.named_parameters():
            if n_.endswith('kernel'):
                p_.mul_(1 + 2.0 ** -16 * torch.randn(p_.shape, generator=g, dtype=torch.float64))
    mg = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV).train()
    o64 = m64(me_cpu.SparseTensor(f.double(), torch.from_numpy(c)))
    opt = mpt(me_cpu.SparseTensor(f.double(), torch.from_numpy(c)))
    og = engine.FusedMinkUNet(mg, batch_stats=True).forward_train(torch.from_numpy(c).to(DEV), f.to(DEV))
    l64, lpt = omatch.distill_loss(o64, tgt.double()), omatch.distill_loss(opt, tgt.double())
    lg = (1 - torch.nn.CosineSimilarity()(og, tgt.to(DEV))).mean()
    assert abs(l64.item() - lg.item()) < max(1e-5, 8 * abs(l64.item() - lpt.item()))
    l64.backward(); lpt.backward(); lg.backward()
    for (n, p64), (_, ppt), (_, pg) in zip(m64.named_parameters(), mpt.named_parameters(), mg.named_parameters()):
        a = p64.grad.numpy()
        e_pert = np.abs(a - ppt.grad.numpy()).max()
        e_gpu = np.abs(a - pg.grad.cpu().numpy().astype(np.float64)).max()
        assert e_gpu <= 10 * e_pert + 1e-3 * np.abs(a).max(), (n, e_gpu, e_pert)
    assert torch.allclose(m64.bn0.bn.running_mean.float(), mg.bn0.bn.running_mean.cpu(), atol=1e-5)
    assert torch.allclose(m64.bn0.bn.running_var.float(), mg.bn0.bn.running_var.cpu(), atol=1e-5)


def test_two_identical_steps_give_identical_gradients_and_stale_graph_raises():
    from openscene_b200 import engine
    c, f = _scene('config1_50k')
    model = synth.build_model('MinkUNet34C', 768, seed=1).to(DEV).train()
    snap = {k: v.clone() for k, v in model.state_dict().items()}
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    mask = (torch.rand(len(c), generator=torch.Generator().manual_seed(3)) < 0.3).to(DEV)
    res = []
    for _ in range(2):
        with torch.no_grad():
            for k, v in model.state_dict().items():
                v.copy_(snap[k])
        model.zero_grad(set_to_none=True)
        out = eng.forward_train(c, f, rows=mask)
        (out * out).sum().backward()
        res.append([p.grad.clone() for p in model.parameters()] + [out.detach().clone()])
    assert all(torch.equal(a, b) for a, b in zip(*res))
    out = eng.forward_train(c, f, rows=mask)
    eng.forward_train(c, f, rows=mask)                     # overwrites what the first graph saved
    with pytest.raises(RuntimeError, match='overwritten'):
        out.sum().backward()
    out = eng.forward_train(c, f, rows=mask)
    with torch.no_grad():
        model.block1[0].conv1.kernel.add_(0.0)             # an in-place weight change: torch's version check
    with pytest.raises(RuntimeError, match='modified by an inplace operation'):
        out.sum().backward()


def test_fused_distill_step_reduces_loss_and_eval_engine_refolds():
    from openscene_b200 import distill, engine
    c = torch.from_numpy(synth.random_cloud(1200, 18, seed=9))
    f = torch.ones(len(c), 3)
    g = torch.Generator().manual_seed(3)
    mask = torch.rand(len(c), generator=g) < 0.6
    tgt = torch.randn(int(mask.sum()), 64, generator=g).half()
    model = synth.build_model('MinkUNet14A', 64, seed=1).to(DEV).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    model.eval()
    eng_eval = engine.FusedMinkUNet(model)
    out0 = eng_eval(c.to(DEV), f.to(DEV)).clone()
    model.train()
    losses = [float(distill.fused_distill_step(eng, opt, c, f, tgt, mask)) for _ in range(6)]
    assert losses[-1] < losses[0] - 0.02, losses
    model.eval()
    out1 = eng_eval(c.to(DEV), f.to(DEV))                  # re-folds the trained weights and moved statistics
    ref = synth.build_model('MinkUNet14A', 64, seed=1)
    ref.load_state_dict(model.state_dict())
    import MinkowskiEngine as ME
    with torch.no_grad():
        r = ref.to(DEV).eval()(ME.SparseTensor(f.to(DEV), c.to(DEV)))
    assert rel_row_err(out1.cpu().numpy(), r.cpu().numpy()) < 1e-3
    assert rel_row_err(out1.cpu().numpy(), out0.cpu().numpy()) > 1e-3


def test_refusals():
    from openscene_b200 import engine
    c, f = _scene('tiny')
    model = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(NotImplementedError, match='input features'):
        eng.forward_train(c, f.clone().requires_grad_())
    model.eval()
    with pytest.raises(RuntimeError, match='train'):
        eng.forward_train(c, f)
    model.train()
    with pytest.raises(RuntimeError, match='batch_stats'):
        engine.FusedMinkUNet(copy.deepcopy(model).eval()).forward_train(c, f)
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
