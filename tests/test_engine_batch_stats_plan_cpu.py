"""Static check of the launch sequence ``FusedMinkUNet(model, batch_stats=True)`` issues, without a GPU.

With batch statistics every BatchNorm needs a full reduction over its layer's output before anything may read it, so the
engine launches each convolution raw (no scale/shift, no ReLU, no residual), reduces the output with ``osb_bn_batch_stats``
and normalises it in place with ``osb_bn_apply_split`` -- except for a BasicBlock's downsample branch, whose raw output is only
reduced and then normalised inside the apply pass of conv2, which reads it as the residual.  An apply that came too late, or a
layer reduced twice (running buffers moved twice), would give results the GPU tests see only for the architectures they run.
Here the engine's own Python runs on CPU tensors with the device entry points recorded (the recorder of
tests/test_engine_plan_cpu.py), for all ten architectures and the scene sizes used there, and the call list is checked."""
import contextlib
import types

import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import engine, minkunet, synth, tc
from tests.test_engine_plan_cpu import HOST_ONLY, SCENES, _FakeCM

_HOST_ONLY = HOST_ONLY | {'osb_bn_stats_workspace_bytes'}


@pytest.fixture
def recorded(monkeypatch):
    """engine + tc running on CPU tensors; device entry points record (name, args) in call order instead of launching"""
    real = C.lib()
    rec = types.SimpleNamespace(calls=[])

    class Lib:
        def __getattr__(self, name):
            if name in _HOST_ONLY:
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
    return rec


def _int(a):
    return 0 if a is None else (a if isinstance(a, int) else a.value or 0)


def _events(calls):
    """call list -> [(kind, dict)] with the pointers as ints"""
    ev = []
    for name, a in calls:
        a = [_int(x) if not isinstance(x, float) else x for x in a]
        if name == 'osb_conv_fwd_tc':
            ev.append(('conv', dict(reads=[a[0], a[3], a[13]], out=a[15], out_f32=a[16], n=a[7], cout=a[10], scale=a[11], shift=a[12],
                                    res=a[13], relu=a[14])))
        elif name == 'osb_convtr_fwd_tc':
            ev.append(('conv', dict(reads=[a[0]], out=a[10], out_f32=a[11], n=None, cout=a[6], scale=a[7], shift=a[8], res=0,
                                    relu=a[9])))
        elif name.startswith('osb_conv_stem_fused'):
            ev.append(('conv', dict(reads=[], out=a[-3], out_f32=_int(a[-2]), n=a[3], cout=a[-7], scale=a[-6], shift=a[-5], res=0,
                                    relu=a[-4])))
        elif name == 'osb_bn_batch_stats':
            ev.append(('stats', dict(x=a[0], n=a[1], c=a[2], w=a[3], b=a[4], eps=a[5], momentum=a[6], rm=a[7], rv=a[8], nbt=a[9],
                                     scale=a[10], shift=a[11], ws=a[12], ws_bytes=a[13])))
        elif name == 'osb_bn_apply_split':
            ev.append(('apply', dict(x=a[0], n=a[1], c=a[2], scale=a[3], shift=a[4], res=a[5], res_scale=a[6], res_shift=a[7],
                                     relu=a[8])))
        elif name in ('osb_gather_rows_f32', 'osb_split_to_f32', 'osb_conv_fwd_f32'):
            ev.append(('other', dict(name=name)))
        else:
            raise AssertionError(f"unexpected entry point {name}")
    return ev


def _bns(model):
    return [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)]


def _n_downsample(eng):
    return sum(ds is not None for (_, blocks) in eng.enc + eng.dec for (_, _, ds) in blocks)


def _check_plan(rec, eng, model, n, out):
    ev = _events(rec.calls)
    convs = [(i, d) for i, (k, d) in enumerate(ev) if k == 'conv']
    stats = [(i, d) for i, (k, d) in enumerate(ev) if k == 'stats']
    applies = [(i, d) for i, (k, d) in enumerate(ev) if k == 'apply']
    bns = _bns(model)

    # ---- every BatchNorm convolution is launched raw; the final one writes fp32 rows in caller order ----------------
    bn_convs, final = convs[:-1], convs[-1][1]
    assert final['out_f32'] == out.data_ptr() and final['out'] == 0 and final['relu'] == 0 and final['scale'] == 0
    assert len(bn_convs) == len(bns)
    for _, d in bn_convs:
        assert d['scale'] == 0 and d['shift'] == 0 and d['relu'] == 0 and d['res'] == 0, d
        assert d['out'] and not d['out_f32']
    outs = [d['out'] for _, d in bn_convs]
    assert len(set(outs)) == len(outs), "two layers write the same activation"
    produced_at = {d['out']: i for i, d in bn_convs}

    # ---- each output is reduced by exactly one osb_bn_batch_stats, after it was written, with its rows and width ----
    stats_of = {}
    for i, s in stats:
        assert s['x'] in produced_at and produced_at[s['x']] < i, "statistics of rows nothing wrote yet"
        assert s['x'] not in stats_of, "a layer's output is reduced twice (its running buffers move twice)"
        stats_of[s['x']] = (i, s)
        assert s['n'] in n and s['n'] >= 2
        assert s['ws'] and s['ws_bytes'] >= C.lib().osb_bn_stats_workspace_bytes(s['n'], s['c'])
    assert set(stats_of) == set(outs)
    for i, d in bn_convs:
        s = stats_of[d['out']][1]
        assert s['c'] == d['cout']
        if d['n'] is not None:
            assert s['n'] == d['n']

    # ---- each BatchNorm module's buffers appear exactly once: one reduction per module and forward --------------------
    rm = [s['rm'] for _, s in stats]
    assert sorted(rm) == sorted(m.running_mean.data_ptr() for m in bns)
    by_rm = {m.running_mean.data_ptr(): m for m in bns}
    for _, s in stats:
        m = by_rm[s['rm']]
        assert (s['rv'], s['nbt'], s['w'], s['b']) == (m.running_var.data_ptr(), m.num_batches_tracked.data_ptr(),
                                                        m.weight.data_ptr(), m.bias.data_ptr())
        assert s['c'] == m.num_features and s['eps'] == m.eps
        assert s['momentum'] == (-1.0 if m.momentum is None else m.momentum)
    slots = sorted((s['scale'], s['shift']) for _, s in stats)
    assert len(set(slots)) == len(slots), "two BatchNorms share a scale / shift slot"

    # ---- applies: after the reduction of the same rows, with its scale / shift; downsample outputs only as residuals --
    applied_at = {}
    for i, a in applies:
        si, s = stats_of[a['x']]
        assert si < i and (a['scale'], a['shift'], a['n'], a['c']) == (s['scale'], s['shift'], s['n'], s['c'])
        assert a['x'] not in applied_at, "rows normalised twice"
        applied_at[a['x']] = i
        assert a['relu'] == 1
        if a['res_scale']:
            ri, rs = stats_of[a['res']]
            assert ri < i, "a downsample's raw output is used as a residual before it was reduced"
            assert (a['res_scale'], a['res_shift']) == (rs['scale'], rs['shift'])
    ds_outs = set(outs) - set(applied_at)
    assert len(ds_outs) == _n_downsample(eng)
    res_norm = [a['res'] for _, a in applies if a['res_scale']]
    assert sorted(res_norm) == sorted(ds_outs), "every downsample output is normalised inside exactly one apply"

    # ---- nothing reads a buffer before it was normalised -------------------------------------------------------------
    for i, (kind, d) in enumerate(ev):
        reads = d['reads'] if kind == 'conv' else ([d['res']] if kind == 'apply' else [])
        for r in reads:
            if not r:
                continue
            assert r in produced_at and produced_at[r] < i
            if r in ds_outs:
                assert kind == 'apply', "a raw downsample output is read by a convolution"
            else:
                assert applied_at[r] < i, f"event {i} ({kind}) reads rows before their BatchNorm was applied"


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_batch_stats_plan(recorded, arch, scene):
    n = SCENES[scene]
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    for _ in range(2):                                              # per forward: every module reduced exactly once
        recorded.calls.clear()
        out = eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=_FakeCM(n))
        assert out.shape == (n[0], 768)
        assert eng._chain_on is False
        _check_plan(recorded, eng, model, n, out)


def test_batch_stats_plan_with_cumulative_momentum(recorded):
    n = SCENES['mid']
    model = synth.build_model('MinkUNet34C', 20, seed=0).train()     # 20-wide head: the generic fp32 final layer
    for m in _bns(model):
        m.momentum = None
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    out = eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=_FakeCM(n))
    ev = _events(recorded.calls)
    assert all(d['momentum'] == -1.0 for k, d in ev if k == 'stats')
    assert len([1 for k, _ in ev if k == 'stats']) == 62


def test_batch_stats_versions_and_no_repack(recorded, monkeypatch):
    """The engine's own running-buffer updates bump the buffers' versions (so eval-mode engines and fast_eval re-fold) but do
    not make the engine itself re-pack; a weight or affine change does."""
    n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    builds = []
    orig = engine.FusedMinkUNet._build
    monkeypatch.setattr(engine.FusedMinkUNet, '_build', lambda self: (builds.append(1), orig(self))[1])
    bn = model.bn0.bn
    v0 = (bn.running_mean._version, bn.running_var._version, bn.num_batches_tracked._version)
    run = lambda: eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=_FakeCM(n))
    run(); run()
    assert builds == []
    v1 = (bn.running_mean._version, bn.running_var._version, bn.num_batches_tracked._version)
    assert all(b > a for a, b in zip(v0, v1))
    with torch.no_grad():
        model.block1[0].norm1.bn.weight.mul_(1.1)
    run()
    assert builds == [1]
    with torch.no_grad():
        model.block2[0].conv1.kernel.add_(0.01)
    run()
    assert builds == [1, 1]
    model.bn1.bn.running_mean = torch.zeros(model.bn1.bn.num_features)     # a re-assigned buffer is re-read
    recorded.calls.clear()
    run()
    assert builds == [1, 1, 1]
    assert model.bn1.bn.running_mean.data_ptr() in [d['rm'] for k, d in _events(recorded.calls) if k == 'stats']


@pytest.mark.parametrize('level', [0, 2, 4])
def test_too_few_rows_refused_before_any_call(recorded, level):
    n = list(SCENES['tiny'])
    n[level] = 1
    for l in range(level + 1, 5):
        n[l] = 1
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    versions = [t._version for t in model.buffers()]
    recorded.calls.clear()
    with pytest.raises(ValueError, match='Expected more than 1 value per channel when training'):
        eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=_FakeCM(n))
    assert recorded.calls == []
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    assert versions == [t._version for t in model.buffers()]


def test_batch_stats_refusals(recorded):
    model = synth.build_model('MinkUNet14A', 64, seed=0)
    with pytest.raises(RuntimeError, match='train'):
        engine.FusedMinkUNet(model.eval(), batch_stats=True)
    with pytest.raises(RuntimeError, match='eval'):
        engine.FusedMinkUNet(model.train())                              # the default still refuses train mode
    model.train()
    model.block1[0].norm1.bn.eval()                                      # a BatchNorm left in eval mode
    with pytest.raises(RuntimeError, match='train'):
        engine.FusedMinkUNet(model, batch_stats=True)
    eng = engine.FusedMinkUNet(synth.build_model('MinkUNet14A', 64, seed=0).train(), batch_stats=True)
    with pytest.raises(NotImplementedError, match='eval-only'):
        eng.fold_head(torch.nn.functional.normalize(torch.randn(4, 64), dim=1))
    with pytest.raises(NotImplementedError, match='eval-only'):
        eng.forward_scores(torch.zeros(4, 4, dtype=torch.int32), torch.ones(4, 3), None)
    eng._net.eval()
    n = SCENES['tiny']
    with pytest.raises(RuntimeError, match='train'):
        eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=_FakeCM(n))
    for attr, value in (('affine', False), ('track_running_stats', False)):
        m = synth.build_model('MinkUNet14A', 64, seed=0).train()
        bn = m.block2[0].norm2.bn
        setattr(bn, attr, value)
        if attr == 'affine':
            bn.weight = bn.bias = None
        else:
            bn.running_mean = bn.running_var = bn.num_batches_tracked = None
        with pytest.raises(NotImplementedError, match='BatchNorm'):
            engine.FusedMinkUNet(m, batch_stats=True)
    m = synth.build_model('MinkUNet14A', 64, seed=0).train()
    m.bn3.bn.running_var = m.bn3.bn.running_var.double()
    with pytest.raises(NotImplementedError, match='fp32'):
        engine.FusedMinkUNet(m, batch_stats=True)
