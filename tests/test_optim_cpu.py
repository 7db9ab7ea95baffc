"""The device optimisers (openscene_b200/optim.py) without a GPU: the engine and the optimiser run on CPU tensors with the device
entry points recorded (the recorder of tests/test_engine_batch_stats_plan_cpu.py), and the tables they would upload decoded.
Checked: the update table's pointers, sizes and per-tensor scalars (torch's double-then-fp32 values), parameters without a
gradient left out and untouched, the re-pack job list against every split-bf16 operand the forward and backward read (for all
ten architectures, each job re-reading its operand's source matrix from the parameter), and the state-dict layout against CPU
``torch.optim.Adam`` / ``SGD``."""
import contextlib
import types

import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import engine, engine_train, minkunet, optim, synth, tc
from tests.test_engine_plan_cpu import HOST_ONLY, SCENES
from tests.test_engine_train_plan_cpu import _CM

_HOST = HOST_ONLY | {'osb_bn_stats_workspace_bytes', 'osb_conv_wgrad_tc_workspace_bytes', 'osb_conv_packed_weight_bytes',
                     'osb_optim_entry_bytes'}


@pytest.fixture
def recorded(monkeypatch):
    real = C.lib()
    rec = types.SimpleNamespace(calls=[], n=None, tables=[], packs={})

    class Lib:
        def __getattr__(self, name):
            if name in _HOST:
                return getattr(real, name)
            return lambda *a: (rec.calls.append((name, a)), 0)[1]

    def pack(w3, transpose_w=False):
        """a zero buffer of the real size, remembering the [K, cout, cin] matrix it stands for"""
        w3 = w3.detach().contiguous().float()
        K = w3.shape[0]
        cin, cout = (w3.shape[2], w3.shape[1]) if transpose_w else (w3.shape[1], w3.shape[2])
        out = torch.zeros(real.osb_conv_packed_weight_bytes(K, cin, cout), dtype=torch.uint8)
        rec.packs[out.data_ptr()] = (w3.clone() if transpose_w else w3.permute(0, 2, 1).clone())
        return out

    def upload(table, device):
        rec.tables.append(table.copy())
        return torch.from_numpy(table.view(np.uint8).copy())

    lib = Lib()
    monkeypatch.setattr(C, 'lib', lambda: lib)
    monkeypatch.setattr(C, 'call', lambda name, *a: rec.calls.append((name, a)))
    monkeypatch.setattr(C, 'require_cuda', lambda t, what: None)
    monkeypatch.setattr(C, 'stream_ptr', lambda: None)
    monkeypatch.setattr(tc, 'pack_weights', pack)
    monkeypatch.setattr(tc, 'pack_weight_tiles', lambda w3, transpose_w=False: torch.zeros(64, dtype=torch.uint8))
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(torch.Tensor, 'record_stream', lambda self, s: None)
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    monkeypatch.setattr(engine_train, 'CoordinateManager', lambda coords, pyramid_levels=0: _CM(rec.n))
    monkeypatch.setattr(optim, '_upload', upload)
    return rec


def _train_once(eng, n):
    out = eng.forward_train(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), rows=torch.arange(n[0]) % 7 == 0)
    out.sum().backward()


def _read_packs(calls):
    """addresses of the split-bf16 operands the recorded launches read"""
    out = set()
    for name, a in calls:
        a = [0 if x is None else (x if isinstance(x, (int, float)) else x.value or 0) for x in a]
        if name == 'osb_conv_fwd_tc':
            out.add(a[9])
        elif name == 'osb_convtr_fwd_tc':
            out.add(a[5])
    return out


def _job_matrix(w, strides, K, cin, cout):
    """the [K, cout, cin] matrix a job reads: element (k, n, c) at w[k sk + n sn + c sc]"""
    base = w._base if w._base is not None else w
    off = (w.data_ptr() - base.data_ptr()) // 4
    return torch.as_strided(base.detach(), (K, cout, cin), strides, off)


@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_repack_jobs_cover_exactly_the_operands_forward_and_backward_read(recorded, arch):
    n = recorded.n = SCENES['tiny']
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    _train_once(eng, n)
    recorded.calls.clear()
    model.zero_grad(set_to_none=True)
    _train_once(eng, n)                                      # the W^T packs exist now: what a step has to refresh
    read = _read_packs(recorded.calls)
    jobs = eng.repack_jobs()
    ptrs = [pk.data_ptr() for (_, pk, *_r) in jobs]
    assert len(ptrs) == len(set(ptrs)), "an operand re-packed twice"
    assert set(ptrs) == read, (len(set(ptrs) - read), len(read - set(ptrs)))
    params = {p.data_ptr() for p in model.parameters()}
    for (w, pk, strides, K, cin, cout, pad) in jobs:
        base = w._base if w._base is not None else w
        assert base.data_ptr() in params
        src = recorded.packs[pk.data_ptr()]                 # what the engine packed into this buffer
        got = _job_matrix(w, strides, K, cin, cout)
        if src.shape[0] == 1 and K > 1:                      # dense-up: [1, K * cout, cin] rows = the job's [K, cout, cin]
            got = got.reshape(1, K * cout, cin)
            assert pad * K <= pk.numel() // (4 * cin)
        assert torch.equal(got, src)
        assert pk.numel() == 4 * K * pad * cin
    table, total = optim.repack_table(jobs)
    assert total == sum(-(-(K * pad * cin) // optim.PACK_CHUNK) for (_, _, _, K, cin, _, pad) in jobs)


def test_bound_step_launches_one_update_and_one_repack_with_the_table_torch_would_compute(recorded):
    n = recorded.n = SCENES['tiny']
    model = synth.build_model('MinkUNet14A', 64, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    params = list(model.parameters())
    head = [p for p in params if p.dim() == 2]
    rest = [p for p in params if p.dim() != 2]
    opt = optim.Adam([{'params': rest}, {'params': head, 'lr': 3e-4}], lr=1e-3)
    opt.bind(eng)
    _train_once(eng, n)
    params[5].grad = None                                   # skipped: no entry, no state, untouched
    for p in params:
        if p.grad is not None:
            p.grad = torch.randn_like(p)                        # real tensors: the addresses the table must carry
    before = params[5].detach().clone()
    refresh = []
    eng.refresh = lambda: refresh.append(1)
    recorded.calls.clear()
    for step in (1, 2):
        opt.param_groups[0]['lr'] = 1e-3 * (1 - step / 10) ** 0.9             # the poly schedule of run/distill.py
        recorded.calls.clear()
        recorded.tables.clear()
        versions = [p._version for p in params]
        opt.step()
        names = [nm for nm, _ in recorded.calls]
        assert names == ['osb_optim_adam', 'osb_conv_repack']
        t = recorded.tables[0]
        want = [(g, p) for g in opt.param_groups for p in g['params'] if p.grad is not None]
        assert len(t) == len(want) == len(params) - 1
        assert recorded.calls[0][1][1:4] == (len(t), optim.OPTIM_CHUNK, int(sum(-(-p.numel() // optim.OPTIM_CHUNK)
                                                                                 for _, p in want)))
        begin = 0
        for r, (g, p) in zip(t, want):
            st = opt.state[p]
            assert (r['param'], r['grad'], r['exp_avg'], r['exp_avg_sq'], r['numel']) == (
                p.data_ptr(), p.grad.data_ptr(), st['exp_avg'].data_ptr(), st['exp_avg_sq'].data_ptr(), p.numel())
            assert r['chunk_begin'] == begin
            begin += -(-p.numel() // optim.OPTIM_CHUNK)
            assert st['step'].dtype == torch.float32 and float(st['step']) == step
            lr, (b1, b2), eps = g['lr'], g['betas'], g['eps']
            want_s = np.array([-(lr / (1 - b1 ** step)), (1 - b2 ** step) ** 0.5, 1 - b1, b2, 1 - b2, eps], dtype=np.float64)
            got = np.array([r[k] for k in ('step_size', 'bc2_sqrt', 'lerp_w', 'beta2', 'one_minus_beta2', 'eps')])
            assert np.array_equal(got.astype(np.float32), want_s.astype(np.float32))
        assert params[5] not in opt.state and torch.equal(params[5], before)
        assert all(p._version > v for p, v in zip(params, versions) if p.grad is not None)
        assert eng._sig == eng._signature()
        assert len(recorded.tables) == (2 if step == 1 else 1)          # the job list did not change: its table stays
    assert refresh == []


def test_sgd_table_first_step_and_momentum_zero(recorded):
    ps = [torch.nn.Parameter(torch.randn(33)), torch.nn.Parameter(torch.randn(4, 5))]
    for p in ps:
        p.grad = torch.randn_like(p)
    opt = optim.SGD([{'params': ps[:1]}, {'params': ps[1:], 'momentum': 0.0}], lr=0.01, momentum=0.9, weight_decay=1e-4)
    for step in (1, 2):
        recorded.tables.clear()
        opt.step()
        t = recorded.tables[0]
        assert t['first'].tolist() == [int(step == 1), 0]
        assert t['momentum_buffer'][0] == opt.state[ps[0]]['momentum_buffer'].data_ptr() and t['momentum_buffer'][1] == 0
        assert 'momentum_buffer' not in opt.state[ps[1]]                  # torch keeps no buffer without momentum
        assert np.array_equal(t['neg_lr'], np.float32([-0.01, -0.01])) and t['momentum'].tolist() == [np.float32(0.9), 0.0]
        assert np.array_equal(t['weight_decay'], np.float32([1e-4, 1e-4]))


@pytest.mark.parametrize('kind', ['adam', 'sgd'])
def test_state_dict_layout_matches_torch(recorded, kind):
    def make(cls):
        ps = [torch.nn.Parameter(torch.randn(7, 3)), torch.nn.Parameter(torch.randn(5))]
        for p in ps:
            p.grad = torch.ones_like(p)
        if kind == 'adam':
            return cls(ps, lr=1e-3)
        return cls(ps, lr=0.01, momentum=0.9, weight_decay=1e-4)
    ours = make(optim.Adam if kind == 'adam' else optim.SGD)
    ref = make(torch.optim.Adam if kind == 'adam' else torch.optim.SGD)
    ours.step()
    with monkeypatch_is_cuda_off():
        ref.step()
    a, b = ours.state_dict(), ref.state_dict()
    assert a['param_groups'] == b['param_groups']
    assert a['state'].keys() == b['state'].keys()
    for i in b['state']:
        assert a['state'][i].keys() == b['state'][i].keys()
        for k, v in b['state'][i].items():
            w = a['state'][i][k]
            assert (w.dtype, w.device, w.shape) == (v.dtype, v.device, v.shape), (k, w, v)
    ref.load_state_dict(a)                                  # ours into torch, torch's into ours
    ours.load_state_dict(b)
    assert ours.state_dict()['param_groups'] == b['param_groups']


@contextlib.contextmanager
def monkeypatch_is_cuda_off():
    """torch's own optimiser must see the CPU tensors as what they are (it picks its CPU path from is_cuda)"""
    saved = torch.Tensor.__dict__['is_cuda']
    del torch.Tensor.is_cuda
    try:
        yield
    finally:
        torch.Tensor.is_cuda = saved


def test_refusals_before_any_launch(recorded):
    p = torch.nn.Parameter(torch.randn(8))
    p.grad = torch.randn(8)
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(weight_decay=1e-4), dict(capturable=True),
               dict(differentiable=True), dict(fused=True), dict(decoupled_weight_decay=True)):
        with pytest.raises(NotImplementedError):
            optim.Adam([p], **kw)
    for kw in (dict(nesterov=True, momentum=0.9), dict(dampening=0.1), dict(maximize=True), dict(fused=True)):
        with pytest.raises(NotImplementedError):
            optim.SGD([p], lr=0.1, **kw)
    opt = optim.Adam([p])
    opt.param_groups[0]['amsgrad'] = True                   # e.g. a torch checkpoint's groups loaded later
    with pytest.raises(NotImplementedError, match='amsgrad'):
        opt.step()
    opt.param_groups[0]['amsgrad'] = False
    for bad in (torch.nn.Parameter(torch.randn(8, dtype=torch.float64)), torch.nn.Parameter(torch.randn(8, 2).t())):
        bad.grad = torch.zeros_like(bad)
        with pytest.raises(NotImplementedError):
            optim.Adam([bad]).step()
    q = torch.nn.Parameter(torch.randn(4, 4))
    q.grad = torch.randn(4, 4).to_sparse()
    with pytest.raises(NotImplementedError, match='sparse'):
        optim.SGD([q], lr=0.1).step()
    with pytest.raises(ValueError, match='batch_stats'):
        optim.Adam(synth.build_model('MinkUNet14A', 64, seed=0).eval().parameters()).bind(
            engine.FusedMinkUNet(synth.build_model('MinkUNet14A', 64, seed=0).eval()))
    model = synth.build_model('MinkUNet14A', 64, seed=0).train()
    with pytest.raises(ValueError, match='not in this optimiser'):
        optim.Adam(list(model.parameters())[1:]).bind(engine.FusedMinkUNet(model, batch_stats=True))
    assert [c for c in recorded.calls if c[0].startswith('osb_optim') or c[0] == 'osb_conv_repack'] == []
    assert len(opt.state[p]) == 0
