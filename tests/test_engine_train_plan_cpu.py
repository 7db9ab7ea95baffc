"""Static check of the launches ``FusedMinkUNet.forward_train`` and its backward issue (openscene_b200/engine_train.py), without a
GPU: the engine's Python runs on CPU tensors with the device entry points recorded (the recorder of
tests/test_engine_batch_stats_plan_cpu.py), for all ten architectures and three scene sizes.  Checked:
  * every BatchNorm is reduced exactly once in forward and once in backward, stage by stage in reverse order;
  * no activation the forward wrote is written again (the backward reads them);
  * every gradient a BatchNorm backward reads holds the contributions of all consumers of that activation;
  * every BatchNorm weight / bias gradient is written by exactly one backward reduce, every kernel gradient by wgrads;
plus a mutated plan as a negative control, the refusals and the stale-graph error."""
import contextlib
import types

import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import engine, engine_train, minkunet, synth, tc
from tests.test_engine_plan_cpu import HOST_ONLY, SCENES, _FakeCM

_HOST = HOST_ONLY | {'osb_bn_stats_workspace_bytes', 'osb_conv_wgrad_tc_workspace_bytes'}


class _CM(_FakeCM):
    def __init__(self, n):
        super().__init__(n)
        self.perm = torch.arange(n[0], dtype=torch.int32)
        self.inv_perm = self.perm.clone()


@pytest.fixture
def recorded(monkeypatch):
    real = C.lib()
    rec = types.SimpleNamespace(calls=[], n=None)

    class Lib:
        def __getattr__(self, name):
            if name in _HOST:
                return getattr(real, name)
            return lambda *a: (rec.calls.append((name, a)), 0)[1]
    lib = Lib()
    monkeypatch.setattr(C, 'lib', lambda: lib)
    monkeypatch.setattr(C, 'call', lambda name, *a: rec.calls.append((name, a)))
    monkeypatch.setattr(C, 'require_cuda', lambda t, what: None)
    monkeypatch.setattr(C, 'stream_ptr', lambda: None)
    monkeypatch.setattr(tc, 'pack_weights', lambda w3, transpose_w=False: torch.zeros(64, dtype=torch.uint8))
    monkeypatch.setattr(tc, 'pack_weight_tiles', lambda w3, transpose_w=False: torch.zeros(64, dtype=torch.uint8))
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(engine_train, 'CoordinateManager', lambda coords, pyramid_levels=0: _CM(rec.n))
    return rec


def _i(a):
    return 0 if a is None else (a if isinstance(a, int) else (a if isinstance(a, float) else (a.value or 0)))


def _ev(name, a):
    """-> (reads, writes, extra) with pointers as ints"""
    a = [_i(x) for x in a]
    if name == 'osb_conv_fwd_tc':
        return [a[0], a[3]], [a[15]], dict(res=a[13], out=a[15])
    if name == 'osb_convtr_fwd_tc':
        return [a[0]], [a[10]], {}
    if name.startswith('osb_conv_stem_fused'):
        return [], [a[-3]], {}
    if name == 'osb_bn_batch_stats_save':
        return [a[0]], [], dict(rm=a[7], mean=a[12])
    if name == 'osb_bn_apply_split_out':
        return [a[0], a[6]], [a[1]], dict(res=a[6], res_scale=a[7])
    if name == 'osb_bn_backward_reduce':
        return [a[0], a[1], a[2]], [], dict(y=a[0], g=a[1], mean=a[5], dw=a[8], db=a[9])
    if name == 'osb_bn_backward_apply':
        return [a[0], a[1], a[2]], [a[9]] + ([a[10]] if a[10] else []), dict(gp=a[10], gp_acc=a[11])
    if name == 'osb_conv_wgrad_tc':
        return [a[0], a[6]], [], dict(gw=a[8])
    if name == 'osb_f32_to_split':
        return [], [a[3]], {}
    return [], [], {}


def _check(calls, nf, model):
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)]
    fwd, bwd = calls[:nf], calls[nf:]
    # forward: one reduction per BatchNorm; record every activation write and every consumer of it
    stats = [_ev(n, a)[2] for n, a in fwd if n == 'osb_bn_batch_stats_save']
    assert sorted(s['rm'] for s in stats) == sorted(m.running_mean.data_ptr() for m in bns)
    written, consumers, stage_of, stage = {}, {}, {}, 0
    for name, a in fwd:
        reads, writes, x = _ev(name, a)
        if name in ('osb_conv_fwd_tc', 'osb_convtr_fwd_tc') and not x.get('res', 0):
            if name == 'osb_convtr_fwd_tc' or a[8] == 8:
                stage += 1
        if name == 'osb_bn_batch_stats_save':
            stage_of[x['mean']] = stage
        for w in writes:
            assert w not in written, "an activation written twice in forward"
            written[w] = True
        srcs = reads if name != 'osb_bn_apply_split_out' else ([x['res']] if x['res'] and not x['res_scale'] else [])
        for r in srcs:
            if r and name != 'osb_bn_batch_stats_save':
                consumers[r] = consumers.get(r, 0) + 1
    # backward
    count, reduced, wgrads, last_stage = {}, [], [], None
    for name, a in bwd:
        reads, writes, x = _ev(name, a)
        for w in writes:
            assert w not in written, "the backward overwrites an activation the forward saved"
        if name == 'osb_conv_fwd_tc':                                  # dgrad: one more contribution on top of `res`
            count[x['out']] = count.get(x['res'], 0) + 1 if x['res'] else 1
        elif name == 'osb_bn_backward_apply' and x['gp']:
            count[x['gp']] = count.get(x['gp'], 0) + 1 if x['gp_acc'] else 1
        elif name == 'osb_bn_backward_reduce':
            assert count.get(x['g'], 0) == consumers[x['y']], "a BatchNorm backward reads an incomplete gradient"
            reduced.append(x)
            s = stage_of[x['mean']]
            assert last_stage is None or s <= last_stage, "the backward does not run the stages in reverse order"
            last_stage = s
        elif name == 'osb_conv_wgrad_tc':
            wgrads.append(x['gw'])
    assert sorted(r['mean'] for r in reduced) == sorted(stage_of), "every BatchNorm reduced once in backward"
    grads = {id(p): p.grad.data_ptr() for p in model.parameters()}
    bn_slots = sorted([r['dw'] for r in reduced] + [r['db'] for r in reduced])
    assert bn_slots == sorted(grads[id(p)] for m in bns for p in (m.weight, m.bias))
    kernels = [m.kernel for m in model.modules() if hasattr(m, 'kernel') and isinstance(m.kernel, torch.nn.Parameter)]
    direct = [g for g in wgrads if g in {grads[id(k)] for k in kernels}]
    assert len(direct) == len(set(direct))
    return len(wgrads)


def _run(eng, n, rows=None):
    return eng.forward_train(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), rows=rows)


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_train_plan(recorded, arch, scene):
    n = recorded.n = SCENES[scene]
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    rows = torch.arange(n[0]) % 7 == 0
    for _ in range(2):
        recorded.calls.clear()
        model.zero_grad(set_to_none=True)
        out = _run(eng, n, rows)
        nf = len(recorded.calls)
        out.sum().backward()
        _check(recorded.calls, nf, model)


def test_mutated_plan_is_caught(recorded):
    """negative control: drop one dgrad that feeds an accumulated gradient"""
    n = recorded.n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    out = _run(eng, n)
    nf = len(recorded.calls)
    out.sum().backward()
    calls = list(recorded.calls)
    i = next(k for k in range(nf, len(calls)) if calls[k][0] == 'osb_conv_fwd_tc' and _ev(*calls[k])[2]['res'])
    res = _ev(*calls[i])[2]['res']
    mutated = calls[:i] + calls[i + 1:]
    # the consumer now reads the chain without the dropped contribution
    mutated = [(nm, a) if nm != 'osb_bn_backward_reduce' or _i(a[1]) != _ev(*calls[i])[2]['out'] else (nm, (a[0], res) + tuple(a[2:]))
               for nm, a in mutated]
    with pytest.raises(AssertionError):
        _check(mutated, nf, model)


def test_refusals_and_stale_graph(recorded):
    n = recorded.n = SCENES['tiny']
    model = synth.build_model('MinkUNet14A', 64, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(NotImplementedError, match='input features'):
        eng.forward_train(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3, requires_grad=True))
    model.eval()
    with pytest.raises(RuntimeError, match='train'):
        _run(eng, n)
    model.train()
    with pytest.raises(RuntimeError, match='batch_stats'):
        _run(engine.FusedMinkUNet(synth.build_model('MinkUNet14A', 64, seed=0).eval()), n)
    small = list(n)
    small[4] = 1
    recorded.n = small
    with pytest.raises(ValueError, match='Expected more than 1 value per channel when training'):
        _run(eng, small)
    assert recorded.calls == []
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    recorded.n = n
    out = _run(eng, n)
    _run(eng, n)                                   # overwrites what the first graph saved
    with pytest.raises(RuntimeError, match='overwritten'):
        out.sum().backward()
    out = _run(eng, n)
    eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=_CM(n))     # a plain forward as well
    with pytest.raises(RuntimeError, match='overwritten'):
        out.sum().backward()
