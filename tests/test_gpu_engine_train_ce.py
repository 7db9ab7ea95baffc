"""``FusedMinkUNet.forward_train_ce`` (run/train_mink.py's step on the fused engine) against the module path and the fp64 oracle
(the kernels themselves: tests/test_gpu_ce_head.py).  Gradients use the perturbed-module-path yardstick of
tests/test_gpu_engine_train.py, for the reason given there (ReLU masks flip under the split-bf16 rounding)."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from openscene_b200 import synth
from tests.test_gpu_engine_train import _Keep, _buffers_close, _grads_close, _perturbed
from tests.util import rel_row_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _labels(coords, c):
    """height bands x x-slabs, mod C, with 10 % of the voxels unlabelled (255): something a network can learn"""
    c64 = coords.long()
    lab = ((c64[:, 3] // 8) * 5 + c64[:, 1] // 16) % c
    lab[(c64[:, 1] * 7 + c64[:, 2] * 13 + c64[:, 3] * 3) % 10 == 0] = 255
    return lab


def _batch(n_scenes, c):
    coords = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=s, batch_index=s)) for s in range(n_scenes)])
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(2))
    return coords.to(DEV), feats.to(DEV), _labels(coords, c).to(DEV)


def _sgd(params):
    return torch.optim.SGD(params, lr=0.01, momentum=0.9, weight_decay=1e-4)      # config/*/mink.yaml


@pytest.mark.parametrize('arch,classes,scenes', [('MinkUNet18A', 20, 4), ('MinkUNet34C', 21, 1)])
def test_fused_step_matches_module_path(arch, classes, scenes):
    from openscene_b200 import engine, train_mink
    c, f, lab = _batch(scenes, classes)
    model = synth.randomize_bn_stats(synth.build_model(arch, classes, seed=3), seed=7).train()
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    m_pt = _perturbed(copy.deepcopy(model).to(DEV))
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    o_mod, o_eng, o_pt = (_Keep(m.parameters(), lr=0.0) for m in (m_mod, m_eng, m_pt))
    logits = []
    m_mod.register_forward_hook(lambda m, i, o: logits.append(o.detach()))
    labelled = lab != 255
    for step in range(3):
        torch.manual_seed(step)
        l_mod, p_mod = train_mink.train_step(m_mod, o_mod, c, f, lab)
        torch.manual_seed(step)
        l_eng, p_eng = train_mink.fused_train_step(eng, o_eng, c, f, lab)
        torch.manual_seed(step)
        train_mink.train_step(m_pt, o_pt, c, f, lab)
        l_mod, l_eng = float(l_mod), float(l_eng)
        print(arch, 'step', step, 'loss', l_mod, l_eng)
        assert abs(l_mod - l_eng) <= 1e-4 * abs(l_mod)
        print('worst grad error / (perturbation + 1e-4 max)', _grads_close(m_eng, m_mod, m_pt))
        _buffers_close(m_eng, m_mod)
        z = logits[-1]
        top2 = z.topk(2, 1).values
        sure = labelled & (top2[:, 0] - top2[:, 1] > 1e-3 * z.abs().max(1).values)
        assert p_eng.dtype == torch.int64 and p_eng.shape == p_mod.shape
        assert torch.equal(p_eng[sure], p_mod[sure])
        agree = float((p_eng == p_mod).float().mean())
        print('pred agreement', agree, 'resolvable labelled rows', float(sure.float().mean()))
        assert agree >= 0.999
    # three real SGD steps from the same weights: the two arms stay together
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    o_mod, o_eng = _sgd(m_mod.parameters()), _sgd(m_eng.parameters())
    for step in range(4):
        l_mod = float(train_mink.train_step(m_mod, o_mod, c, f, lab, translate=False)[0])
        l_eng = float(train_mink.fused_train_step(eng, o_eng, c, f, lab, translate=False)[0])
        print(arch, 'SGD step', step, l_mod, l_eng)
        assert abs(l_mod - l_eng) <= 1e-3 * abs(l_mod)


def test_against_fp64_oracle():
    """the yardstick of test_gpu_engine_train.py::test_against_fp64_oracle"""
    from openscene_b200 import engine
    from oracle import me_cpu
    c = synth.scene('tiny')
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(0))
    lab = _labels(torch.from_numpy(c), 20)
    m64 = synth.build_model('MinkUNet14A', 20, seed=0, ME=me_cpu.as_module()).double().train()
    mpt = copy.deepcopy(m64)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n_, p_ in mpt.named_parameters():
            if n_.endswith('kernel'):
                p_.mul_(1 + 2.0 ** -16 * torch.randn(p_.shape, generator=g, dtype=torch.float64))
    mg = synth.build_model('MinkUNet14A', 20, seed=0).to(DEV).train()
    l64 = F.cross_entropy(m64(me_cpu.SparseTensor(f.double(), torch.from_numpy(c))), lab, ignore_index=255)
    lpt = F.cross_entropy(mpt(me_cpu.SparseTensor(f.double(), torch.from_numpy(c))), lab, ignore_index=255)
    lg, _ = engine.FusedMinkUNet(mg, batch_stats=True).forward_train_ce(torch.from_numpy(c).to(DEV), f.to(DEV), lab.to(DEV),
                                                                        ignore_index=255)
    assert abs(l64.item() - lg.item()) < max(1e-5, 8 * abs(l64.item() - lpt.item()))
    l64.backward(); lpt.backward(); lg.backward()
    for (n, p64), (_, ppt), (_, pg) in zip(m64.named_parameters(), mpt.named_parameters(), mg.named_parameters()):
        a = p64.grad.numpy()
        e_pert = np.abs(a - ppt.grad.numpy()).max()
        e_gpu = np.abs(a - pg.grad.cpu().numpy().astype(np.float64)).max()
        assert e_gpu <= 10 * e_pert + 1e-3 * np.abs(a).max(), (n, e_gpu, e_pert)
    assert torch.allclose(m64.bn0.bn.running_mean.float(), mg.bn0.bn.running_mean.cpu(), atol=1e-5)
    assert torch.allclose(m64.bn0.bn.running_var.float(), mg.bn0.bn.running_var.cpu(), atol=1e-5)


def test_two_identical_steps_are_bit_identical():
    from openscene_b200 import engine
    c, f, lab = _batch(1, 20)
    model = synth.build_model('MinkUNet34C', 20, seed=1).to(DEV).train()
    snap = {k: v.clone() for k, v in model.state_dict().items()}
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    res = []
    for _ in range(2):
        with torch.no_grad():
            for k, v in model.state_dict().items():
                v.copy_(snap[k])
        model.zero_grad(set_to_none=True)
        loss, pred = eng.forward_train_ce(c, f, lab.int(), ignore_index=255)
        loss.backward()
        res.append([p.grad.clone() for p in model.parameters()] + [loss.detach().clone(), pred.clone()])
    assert all(torch.equal(a, b) for a, b in zip(*res))


def test_fused_train_step_reduces_loss_and_eval_engine_refolds():
    from openscene_b200 import engine, train_mink
    import MinkowskiEngine as ME
    c = torch.from_numpy(synth.random_cloud(1200, 18, seed=9))
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(4))
    lab = ((c[:, 3].long() // 6) * 3 + c[:, 1].long() // 6) % 20
    model = synth.build_model('MinkUNet14A', 20, seed=1).to(DEV).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = _sgd(model.parameters())
    losses = [float(train_mink.fused_train_step(eng, opt, c, f, lab)[0]) for _ in range(6)]
    assert losses[-1] < losses[0] - 0.02, losses
    model.eval()
    out = engine.FusedMinkUNet(model)(c.to(DEV), f.to(DEV))            # re-folds the trained weights and moved statistics
    ref = synth.build_model('MinkUNet14A', 20, seed=1)
    ref.load_state_dict(model.state_dict())
    with torch.no_grad():
        r = ref.to(DEV).eval()(ME.SparseTensor(f.to(DEV), c.to(DEV)))
    assert rel_row_err(out.cpu().numpy(), r.cpu().numpy()) < 1e-3


def test_all_ignored_batch():
    from openscene_b200 import engine, train_mink
    c, f, _ = _batch(1, 20)
    lab = torch.full((len(c),), 255, dtype=torch.int64, device=DEV)
    model = synth.build_model('MinkUNet18A', 20, seed=2).train()
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    l_mod, _ = train_mink.train_step(m_mod, _Keep(m_mod.parameters(), lr=0.0), c, f, lab, translate=False)
    l_eng, _ = train_mink.fused_train_step(eng, _Keep(m_eng.parameters(), lr=0.0), c, f, lab, translate=False)
    assert torch.isnan(l_mod) and torch.isnan(l_eng)
    for p in m_eng.parameters():
        assert torch.count_nonzero(p.grad) == 0
    _buffers_close(m_eng, m_mod)


def test_refusals_and_stale_graph():
    from openscene_b200 import engine
    c, f, _ = _batch(1, 20)
    c, f = c[:3000], f[:3000]
    lab = _labels(c.cpu(), 20).to(DEV)
    model = synth.build_model('MinkUNet14A', 20, seed=0).to(DEV).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(NotImplementedError, match='input features'):
        eng.forward_train_ce(c, f.clone().requires_grad_(), lab, 255)
    with pytest.raises(ValueError, match=r'\[N\]'):
        eng.forward_train_ce(c, f, lab[1:], 255)
    with pytest.raises(TypeError, match='integer'):
        eng.forward_train_ce(c, f, lab.float(), 255)
    bad = lab.clone()
    bad[5] = 20
    with pytest.raises(IndexError, match='out of bounds'):
        eng.forward_train_ce(c, f, bad, 255)
    with pytest.raises(NotImplementedError, match='forward_train_ce'):
        eng.forward_train(c, f)
    model.eval()
    with pytest.raises(RuntimeError, match='train'):
        eng.forward_train_ce(c, f, lab, 255)
    model.train()
    with pytest.raises(RuntimeError, match='batch_stats'):
        engine.FusedMinkUNet(copy.deepcopy(model).eval()).forward_train_ce(c, f, lab, 255)
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    loss, _ = eng.forward_train_ce(c, f, lab.to(torch.uint8), 255)          # uint8 labels are widened
    eng.forward_train_ce(c, f, lab, 255)                                    # overwrites what the first graph saved
    with pytest.raises(RuntimeError, match='overwritten'):
        loss.backward()
