"""Static check of the launches ``FusedMinkUNet.forward_train_ce`` and its backward issue (openscene_b200/engine_train.py),
without a GPU: the recorder and ``_check`` of tests/test_engine_train_plan_cpu.py, taught the two cross-entropy entry points,
for all ten architectures and three scene sizes with heads of 16, 20 and 21 classes (and one of 64).  Checked, on top of what
``_check`` checks (every BatchNorm reduced once forward and once backward in reverse stage order, no saved activation
overwritten, every gradient complete before a BatchNorm backward reads it):
  * the backward starts with osb_ce_head_bwd, which alone writes ``final.kernel``'s gradient slot and the trunk's gradient;
  * no tensor-core head launch and no W^T pack of the head;
plus a mutated plan as a negative control, the refusals (nothing recorded, state dict unchanged) and the stale-graph error."""
import pytest
import torch

from openscene_b200 import engine, minkunet, synth
from tests import test_engine_train_plan_cpu as tp
from tests.test_engine_plan_cpu import SCENES
from tests.test_engine_train_plan_cpu import recorded  # noqa: F401  (fixture)

_base_ev = tp._ev


def _ev(name, a):
    if name == 'osb_ce_head_fwd':
        a = [tp._i(x) for x in a]
        return [a[0]], [a[9], a[10]], dict(x=a[0], lse=a[9])
    if name == 'osb_ce_head_bwd':
        a = [tp._i(x) for x in a]
        return [a[0], a[9]], [a[12]], dict(x=a[0], lse=a[9], dx=a[12], dw=a[13])
    return _base_ev(name, a)


@pytest.fixture
def rec(recorded, monkeypatch):  # noqa: F811
    monkeypatch.setattr(tp, '_ev', _ev)
    monkeypatch.setattr(tp, '_HOST', tp._HOST | {'osb_ce_head_workspace_bytes'})
    return recorded


def _as_dgrad(calls):
    """_check counts gradient contributions of dgrads: the CE backward enters it as the one dgrad writing the trunk's gradient"""
    out = []
    for name, a in calls:
        if name == 'osb_ce_head_bwd':
            fake = [0] * 22
            fake[15] = tp._i(a[12])
            out.append(('osb_conv_fwd_tc', tuple(fake)))
        else:
            out.append((name, a))
    return out


def _labels(n0, c, ignore=255):
    lab = torch.arange(n0) % c
    lab[torch.arange(n0) % 10 == 3] = ignore
    return lab


def _run(eng, n, labels, ignore=255, feats=None):
    f = torch.ones(n[0], 3) if feats is None else feats
    return eng.forward_train_ce(torch.zeros(n[0], 4, dtype=torch.int32), f, labels, ignore_index=ignore)


def _check_ce(calls, nf, model, eng):
    tp._check(_as_dgrad(calls), nf, model)
    fwd, bwd = calls[:nf], calls[nf:]
    ce_f = [a for n_, a in fwd if n_ == 'osb_ce_head_fwd']
    ce_b = [a for n_, a in bwd if n_ == 'osb_ce_head_bwd']
    assert len(ce_f) == 1 and len(ce_b) == 1 and bwd[0][0] == 'osb_ce_head_bwd', "the backward starts from the CE head"
    xf, xb = _ev('osb_ce_head_fwd', ce_f[0])[2], _ev('osb_ce_head_bwd', ce_b[0])[2]
    assert xb['x'] == xf['x'] and xb['lse'] == xf['lse']
    gk = model.final.kernel.grad.data_ptr()
    assert xb['dw'] == gk
    assert not any(_ev(n_, a)[2].get('gw') == gk for n_, a in bwd if n_ == 'osb_conv_wgrad_tc'), "final.kernel written twice"
    # no tensor-core head: no convolution writes fp32 rows, no head map transposed, no W^T of the head
    assert not any(n_ == 'osb_conv_fwd_tc' and tp._i(a[16]) for n_, a in calls)
    assert not any(n_ == 'osb_kernel_map_transpose' for n_, a in fwd)
    assert not isinstance(eng.final.bwd, list)


def _step(rec, eng, model, n, labels):
    rec.calls.clear()
    model.zero_grad(set_to_none=True)
    loss, pred = _run(eng, n, labels)
    nf = len(rec.calls)
    assert loss.dim() == 0 and loss.grad_fn is not None and pred.shape == (n[0],) and pred.dtype == torch.int64
    loss.backward()
    _check_ce(rec.calls, nf, model, eng)


@pytest.mark.parametrize('classes', [16, 20, 21])
@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_train_ce_plan(rec, arch, scene, classes):
    n = rec.n = SCENES[scene]
    model = synth.build_model(arch, classes, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    for _ in range(2):
        _step(rec, eng, model, n, _labels(n[0], classes))


def test_train_ce_plan_head_of_64(rec):
    """a head whose width the tensor-core kernels would take still runs through the CE kernels"""
    n = rec.n = SCENES['mid']
    model = synth.build_model('MinkUNet34C', 64, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    _step(rec, eng, model, n, _labels(n[0], 64).int())


def test_mutated_ce_plan_is_caught(rec):
    """negative control: without the CE backward the trunk's gradient is never written"""
    n = rec.n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 20, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    loss, _ = _run(eng, n, _labels(n[0], 20))
    nf = len(rec.calls)
    loss.backward()
    calls = list(rec.calls)
    _check_ce(calls, nf, model, eng)
    mutated = [(nm, a) for nm, a in calls if nm != 'osb_ce_head_bwd']
    with pytest.raises(AssertionError):
        tp._check(_as_dgrad(mutated), nf, model)


def test_ce_refusals_and_stale_graph(rec):
    n = rec.n = SCENES['tiny']
    model = synth.build_model('MinkUNet14A', 20, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    lab = _labels(n[0], 20)
    with pytest.raises(NotImplementedError, match='input features'):
        _run(eng, n, lab, feats=torch.ones(n[0], 3, requires_grad=True))
    with pytest.raises(ValueError, match=r'\[N\]'):
        _run(eng, n, lab[:-1])
    with pytest.raises(ValueError, match=r'\[N\]'):
        _run(eng, n, lab.view(-1, 1))
    with pytest.raises(TypeError, match='integer'):
        _run(eng, n, lab.float())
    with pytest.raises(TypeError, match='integer'):
        _run(eng, n, lab > 3)
    bad = lab.clone()
    bad[7] = 20
    with pytest.raises(IndexError, match='out of bounds'):
        _run(eng, n, bad)
    bad[7] = -1
    with pytest.raises(IndexError, match='out of bounds'):
        _run(eng, n, bad)
    with pytest.raises(IndexError, match='out of bounds'):           # 255 is a class index when ignore_index is -100
        _run(eng, n, lab, ignore=-100)
    model.eval()
    with pytest.raises(RuntimeError, match='train'):
        _run(eng, n, lab)
    model.train()
    with pytest.raises(RuntimeError, match='batch_stats'):
        _run(engine.FusedMinkUNet(synth.build_model('MinkUNet14A', 20, seed=0).eval()), n, lab)
    wide = synth.build_model('MinkUNet14A', 161, seed=0).train()
    with pytest.raises(NotImplementedError, match='161'):
        _run(engine.FusedMinkUNet(wide, batch_stats=True), n, torch.zeros(n[0], dtype=torch.int64))
    small = list(n)
    small[4] = 1
    rec.n = small
    with pytest.raises(ValueError, match='Expected more than 1 value per channel when training'):
        _run(eng, small, lab)
    assert rec.calls == []
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    rec.n = n
    _run(eng, n, lab.to(torch.uint8))                                  # uint8 labels are widened, not refused
    loss, _ = _run(eng, n, lab)
    _run(eng, n, lab)                                                  # overwrites what the first graph saved
    with pytest.raises(RuntimeError, match='overwritten'):
        loss.backward()
    loss, _ = _run(eng, n, lab)
    eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=tp._CM(n))
    with pytest.raises(RuntimeError, match='overwritten'):
        loss.backward()
