"""Static check of the launches ``FusedMinkUNet.forward_train_l1`` and its backward issue (openscene_b200/engine_train.py),
without a GPU: the recorder and ``_check`` of tests/test_engine_train_plan_cpu.py, taught the two L1-head entry points, for
all ten architectures and three scene sizes with heads of 512 and 768 channels.  Checked, on top of what ``_check`` checks:
  * the L1 plan is the cosine plan (tests/test_engine_train_cos_plan_cpu.py) with the head's two entry points swapped;
  * the backward starts with osb_l1_head_bwd, which reads the signs the forward wrote and alone writes ``final.kernel``'s
    gradient slot and the trunk's gradient;
  * no tensor-core head launch, no fp32 -> split conversion of a head gradient and no W^T pack of the head;
  * the PDL window rule of tests/launch_order.py holds on the L1 plan;
plus a mutated plan as a negative control, the refusals (nothing recorded, state dict unchanged) and the stale-graph error."""
import pytest
import torch

from openscene_b200 import distill, engine, engine_train, minkunet, synth
from tests import launch_order as LO
from tests import test_engine_train_cos_plan_cpu as _cp
from tests import test_engine_train_plan_cpu as tp
from tests.test_engine_plan_cpu import SCENES
from tests.test_engine_train_plan_cpu import recorded  # noqa: F401  (fixture)
from tests.test_engine_train_plan_cpu import recorded as train_recorded  # noqa: F401  (fixture)

def _ev(name, a):
    if name == 'osb_l1_head_fwd':
        a = [tp._i(x) for x in a]
        return [a[0]], [a[8]], dict(x=a[0], rows=a[5], target=a[7], signs=a[8])
    if name == 'osb_l1_head_bwd':
        a = [tp._i(x) for x in a]
        return [a[0], a[7]], [a[9]], dict(x=a[0], rows=a[5], signs=a[7], g=a[8], dx=a[9], dw=a[10])
    return _cp._ev(name, a)


@pytest.fixture
def rec(recorded, monkeypatch):  # noqa: F811
    monkeypatch.setattr(tp, '_ev', _ev)
    monkeypatch.setattr(tp, '_HOST', tp._HOST | {'osb_l1_head_workspace_bytes', 'osb_cos_head_workspace_bytes'})
    return recorded


def _as_dgrad(calls):
    """_check counts gradient contributions of dgrads: the L1 backward enters it as the one dgrad writing the trunk's
    gradient"""
    out = []
    for name, a in calls:
        if name == 'osb_l1_head_bwd':
            fake = [0] * 22
            fake[15] = tp._i(a[9])
            out.append(('osb_conv_fwd_tc', tuple(fake)))
        else:
            out.append((name, a))
    return out


def _target(m, c):
    return torch.ones(m, c, dtype=torch.float16)


def _run(eng, n, rows, target, feats=None):
    f = torch.ones(n[0], 3) if feats is None else feats
    return eng.forward_train_l1(torch.zeros(n[0], 4, dtype=torch.int32), f, target, rows)


def _check_l1(calls, nf, model, eng):
    tp._check(_as_dgrad(calls), nf, model)
    fwd, bwd = calls[:nf], calls[nf:]
    cf = [a for n_, a in fwd if n_ == 'osb_l1_head_fwd']
    cb = [a for n_, a in bwd if n_ == 'osb_l1_head_bwd']
    assert len(cf) == 1 and len(cb) == 1 and bwd[0][0] == 'osb_l1_head_bwd', "the backward starts from the L1 head"
    xf, xb = _ev('osb_l1_head_fwd', cf[0])[2], _ev('osb_l1_head_bwd', cb[0])[2]
    assert xb['x'] == xf['x'] and xb['rows'] == xf['rows'] and xb['signs'] == xf['signs']
    gk = model.final.kernel.grad.data_ptr()
    assert xb['dw'] == gk
    assert not any(_ev(n_, a)[2].get('gw') == gk for n_, a in bwd if n_ == 'osb_conv_wgrad_tc'), "final.kernel written twice"
    # no tensor-core head: no convolution writes fp32 rows, no head map transposed, no split conversion of a C-wide gradient,
    # no W^T of the head
    assert not any(n_ == 'osb_conv_fwd_tc' and tp._i(a[16]) for n_, a in calls)
    assert not any(n_ == 'osb_kernel_map_transpose' for n_, a in fwd)
    assert not any(n_ == 'osb_f32_to_split' and tp._i(a[2]) == model.final.kernel.shape[1] for n_, a in bwd)
    assert not isinstance(eng.final.bwd, list)


@pytest.mark.parametrize('width', [512, 768])
@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_train_l1_plan(rec, arch, scene, width):
    n = rec.n = SCENES[scene]
    model = synth.build_model(arch, width, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    rows = torch.arange(n[0]) % 7 == 0
    for _ in range(2):
        rec.calls.clear()
        model.zero_grad(set_to_none=True)
        loss = _run(eng, n, rows, _target(int(rows.sum()), width))
        nf = len(rec.calls)
        assert loss.dim() == 0 and loss.dtype == torch.float32 and loss.grad_fn is not None
        loss.backward()
        _check_l1(rec.calls, nf, model, eng)
        l1_names = [nm for nm, _ in rec.calls]
    # the cosine plan on the same engine, the head's entry points swapped, is the same launch sequence
    rec.calls.clear()
    model.zero_grad(set_to_none=True)
    loss = eng.forward_train_cosine(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), _target(int(rows.sum()),
                                                                                                         width), rows)
    loss.backward()
    swap = {'osb_cos_head_fwd': 'osb_l1_head_fwd', 'osb_cos_head_bwd': 'osb_l1_head_bwd'}
    assert [swap.get(nm, nm) for nm, _ in rec.calls] == l1_names


def test_l1_plan_int64_rows_and_bucket_plan(rec):
    """an int64 row index reaches the head as the selected rows; the all-reduce buckets and the tape items they are due
    after are those of forward_train's tape (DistributedDataParallel's buckets, the head's backward one item)"""
    from openscene_b200 import engine_train
    n = rec.n = SCENES['mid']
    model = synth.build_model('MinkUNet34C', 512, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    idx = torch.arange(0, n[0], 5)
    loss = _run(eng, n, idx, _target(idx.numel(), 512))
    nf = len(rec.calls)
    fwd = [a for n_, a in rec.calls[:nf] if n_ == 'osb_l1_head_fwd']
    assert tp._i(fwd[0][6]) == idx.numel()
    loss.backward()
    _check_l1(rec.calls, nf, model, eng)
    params = list(model.parameters())
    graph = engine_train._run_forward(eng, torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), idx,
                                      l1=_target(idx.numel(), 512))
    buckets = engine_train.plan_buckets(graph.tape, params)
    plain = engine_train._run_forward(eng, torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), idx)
    assert [k for k, _ in graph.tape][:-1] == [k for k, _ in plain.tape][:-1] and graph.tape[-1][0] == 'l1_head'
    assert buckets == engine_train.plan_buckets(plain.tape, params)
    assert buckets[0][1] == len(params) and buckets[-1][0] == 0


def test_mutated_l1_plan_is_caught(rec):
    """negative control: without the L1 backward the trunk's gradient is never written"""
    n = rec.n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    rows = torch.arange(n[0]) % 3 == 0
    loss = _run(eng, n, rows, _target(int(rows.sum()), 768))
    nf = len(rec.calls)
    loss.backward()
    calls = list(rec.calls)
    _check_l1(calls, nf, model, eng)
    mutated = [(nm, a) for nm, a in calls if nm != 'osb_l1_head_bwd']
    with pytest.raises(AssertionError):
        tp._check(_as_dgrad(mutated), nf, model)


def test_l1_refusals_and_stale_graph(rec):
    n = rec.n = SCENES['tiny']
    model = synth.build_model('MinkUNet14A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    rows = torch.arange(n[0]) % 4 == 1
    m = int(rows.sum())
    tgt = _target(m, 768)
    with pytest.raises(NotImplementedError, match='input features'):
        _run(eng, n, rows, tgt, feats=torch.ones(n[0], 3, requires_grad=True))
    with pytest.raises(ValueError, match='no rows'):
        _run(eng, n, torch.zeros(n[0], dtype=torch.bool), _target(0, 768))
    with pytest.raises(ValueError, match='repeated'):
        _run(eng, n, torch.tensor([3, 5, 3]), _target(3, 768))
    with pytest.raises(ValueError, match='mask of shape'):
        _run(eng, n, rows[:-1], tgt)
    with pytest.raises(TypeError, match='fp16'):
        _run(eng, n, rows, tgt.float())
    with pytest.raises(ValueError, match=r'\[M, 768\]'):
        _run(eng, n, rows, _target(m, 512))
    with pytest.raises(ValueError, match='rows for'):
        _run(eng, n, rows, _target(m + 1, 768))
    with pytest.raises(ValueError, match='is on'):
        _run(eng, n, rows, tgt.to('meta'))
    model.eval()
    with pytest.raises(RuntimeError, match='train'):
        _run(eng, n, rows, tgt)
    model.train()
    with pytest.raises(RuntimeError, match='batch_stats'):
        _run(engine.FusedMinkUNet(synth.build_model('MinkUNet14A', 768, seed=0).eval()), n, rows, tgt)
    for width in (96, 640):
        odd = synth.build_model('MinkUNet14A', width, seed=0).train()
        with pytest.raises(NotImplementedError, match='forward_train and distill_loss'):
            _run(engine.FusedMinkUNet(odd, batch_stats=True), n, rows, _target(m, width))
    assert rec.calls == []
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    loss = _run(eng, n, rows, tgt)
    _run(eng, n, rows, tgt)                                            # overwrites what the first graph saved
    with pytest.raises(RuntimeError, match='overwritten'):
        loss.backward()
    loss = _run(eng, n, rows, tgt)
    eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=tp._CM(n))
    with pytest.raises(RuntimeError, match='overwritten'):
        loss.backward()


def test_fused_l1_step_runs_the_l1_head(rec):
    n = rec.n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 512, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    mask = torch.arange(n[0]) % 2 == 0
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    distill.fused_l1_step(eng, opt, torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3),
                              torch.ones(int(mask.sum()), 512), mask)
    names = [nm for nm, _ in rec.calls]
    assert names.count('osb_l1_head_fwd') == 1 and names.count('osb_l1_head_bwd') == 1


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_l1_plan_respects_pdl_windows(train_recorded, monkeypatch, arch, scene):  # noqa: F811
    from tests import test_launch_order_cpu as lo
    assert LO.is_host_only('osb_l1_head_workspace_bytes')
    monkeypatch.setattr(tp, '_HOST', tp._HOST | {'osb_l1_head_workspace_bytes'})
    n = train_recorded.n = SCENES[scene]
    monkeypatch.setattr(engine_train, 'CoordinateManager', lambda coords, pyramid_levels=0: lo._SizedCM(n))
    seq = lo._in_order(monkeypatch)
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    rows = torch.arange(n[0]) % 7 == 0
    target = torch.ones(int(rows.sum()), 768, dtype=torch.float16)
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        loss = eng.forward_train_l1(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), target, rows)
        (0.75 * loss).backward()
    s = lo._summary(seq)
    assert not s['bad'], s['bad'][:3]
    assert s['pdl'] > 0 and s['windows'] == s['pdl']
    heads = [L for L in seq if L.name in ('osb_l1_head_fwd', 'osb_l1_head_bwd')]
    assert [L.name for L in heads] == ['osb_l1_head_fwd', 'osb_l1_head_bwd'] * 2 and not any(L.pdl or L.triggers for L in heads)
    assert not any(L.name == 'osb_conv_fwd_tc' and L.writes and any(w[2] == 'out_f32' for w in L.writes) for L in seq)
