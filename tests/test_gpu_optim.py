"""The device optimisers (openscene_b200/optim.py, csrc/optim.cu) on the GPU.

1. the update kernels bit for bit against tests/optim_ref.py, within fp64 bounds (as torch.optim's foreach updates), with
   torch's NaN positions, over odd sizes, unaligned views, two groups, steps 1 / 2 / 1000 and special gradients;
2. the in-place re-pack: every pack keeps its address and equals a fresh pack; no refresh(); the next forward and backward
   equal a freshly built engine's, bit for bit;
3. five training steps of fused_distill_step (Adam) and fused_train_step (SGD) against torch.optim;
4. checkpoints between these optimisers and torch's, and an interrupted run equal to an uninterrupted one;
5. other consumers of the same parameters (eval engine, fast_eval, module path) see the write;
6. a bound step costs two library launches whatever the parameter count; 7. refusals launch nothing."""
import copy
import io

import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import engine, optim, synth, tc
from tests import optim_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

SIZES = [1, 3, 4, 5, 31, 32, 33, 4097, 2 ** 20 + 3]
SPECIAL = [0.0, -0.0, 1e-40, -1e-42, 1e-45, 1e38, -3e38, float('nan'), float('inf'), -float('inf')]


def _bits(t):
    """fp32 bits, every NaN as 0x7FC00000: the device writes 0x7FFFFFFF for an invalid operation, NumPy 0x7FC00000 or
    0xFFC00000; NaN positions are compared on their own"""
    return _canon(t.detach().float().contiguous().cpu().numpy())


def _canon(a):
    a = np.asarray(a, dtype=np.float32).reshape(-1)
    return np.where(np.isnan(a), np.uint32(0x7FC00000), a.view(np.uint32))


def _params(seed):
    """parameters of every size, as views at odd offsets into bigger storages, plus a [125, 3, 32] kernel; their grads
    views at other offsets, with the special values sprinkled in"""
    g = torch.Generator().manual_seed(seed)
    ps = []
    for i, n in enumerate(SIZES + [(125, 3, 32)]):
        shape = (n,) if isinstance(n, int) else n
        numel = int(np.prod(shape))
        off = i % 4                                               # 0 = aligned; 1..3 = every float4 phase
        base = torch.randn(numel + 4, generator=g).to(DEV)
        p = torch.nn.Parameter(base[off:off + numel].view(shape))
        gb = (torch.randn(numel + 4, generator=g) * 10.0 ** float(torch.randint(-3, 3, (1,), generator=g))).to(DEV)
        goff = (off + 1 + i) % 4
        gr = gb[goff:goff + numel].view(shape)
        k = min(numel, len(SPECIAL))
        idx = torch.randperm(numel, generator=g)[:k].to(DEV)
        gr.view(-1)[idx] = torch.tensor(SPECIAL[:k], dtype=torch.float32, device=DEV)
        p.grad = gr
        ps.append(p)
    return ps


def _clone_params(ps):
    out = []
    for p in ps:
        q = torch.nn.Parameter(p.detach().clone())
        q.grad = p.grad.clone()
        out.append(q)
    return out


def _check(name, mine, ref, p64, bound, theirs):
    """ours == optim_ref bit for bit; finite results (ours and torch's) within the fp64 bound; NaN where torch has NaN"""
    a, r, t = _bits(mine), _canon(ref), _bits(theirs)
    assert np.array_equal(a, r), f"{name}: {int((a != r).sum())} elements differ from optim_ref"
    af, tf = a.view(np.float32), t.view(np.float32)        # NaNs canonical: payloads aside
    p64, bound = p64.reshape(-1), bound.reshape(-1)
    fin = np.isfinite(p64) & np.isfinite(af)
    with np.errstate(all='ignore'):
        assert np.all(np.abs(af[fin].astype(np.float64) - p64[fin]) <= bound[fin]), name
        tfin = np.isfinite(p64) & np.isfinite(tf)
        assert np.all(np.abs(tf[tfin].astype(np.float64) - p64[tfin]) <= bound[tfin]), f"{name}: torch outside the bound"
    assert np.array_equal(np.isnan(af), np.isnan(tf)), f"{name}: NaN positions differ from torch's"
    return int((a == t).sum()), a.size


@pytest.mark.parametrize('step', [1, 2, 1000])
def test_adam_update_arithmetic(step):
    ps = _params(step)
    tp = _clone_params(ps)
    groups = lambda q: [{'params': q[:6]}, {'params': q[6:], 'lr': 3e-4}]
    ours, theirs = optim.Adam(groups(ps), lr=1e-3), torch.optim.Adam(groups(tp), lr=1e-3, foreach=True)
    g = torch.Generator().manual_seed(100 + step)
    if step > 1:                                             # the state a run would have reached
        for p, q in zip(ps, tp):
            m = torch.randn(p.shape, generator=g).to(DEV) * 1e-2
            v = torch.rand(p.shape, generator=g).to(DEV) * 1e-3
            for opt, x in ((ours, p), (theirs, q)):
                opt.state[x] = {'step': torch.tensor(float(step - 1)), 'exp_avg': m.clone(), 'exp_avg_sq': v.clone()}
    before = [(p.detach().cpu().numpy().copy(), p.grad.cpu().numpy().copy(),
               ours.state[p]['exp_avg'].cpu().numpy().copy() if step > 1 else np.zeros(p.shape, np.float32),
               ours.state[p]['exp_avg_sq'].cpu().numpy().copy() if step > 1 else np.zeros(p.shape, np.float32)) for p in ps]
    ours.step()
    theirs.step()
    torch.cuda.synchronize()
    eq = tot = 0
    for i, (p, q) in enumerate(zip(ps, tp)):
        grp = ours.param_groups[0 if i < 6 else 1]
        lr, (b1, b2), eps = grp['lr'], grp['betas'], grp['eps']
        assert float(ours.state[p]['step']) == float(theirs.state[q]['step']) == step
        s = (-(lr / (1 - b1 ** step)), (1 - b2 ** step) ** 0.5, 1 - b1, b2, 1 - b2, eps)
        p0, g0, m0, v0 = before[i]
        rp, rm, rv = R.adam(p0, g0, m0, v0, *s)
        p64, bound = R.adam_bound(p0, g0, m0, v0, *s)
        e, n = _check(f"param {i}", p, rp, p64, bound, q)
        eq, tot = eq + e, tot + n
        assert np.array_equal(_bits(ours.state[p]['exp_avg']), _canon(rm))
        assert np.array_equal(_bits(ours.state[p]['exp_avg_sq']), _canon(rv))
        for k in ('exp_avg', 'exp_avg_sq'):
            a, t = _bits(ours.state[p][k]), _bits(theirs.state[q][k])
            print(f"step {step} param {i} {k}: bit-equal to torch {float((a == t).mean()):.6f}")
    print(f"Adam step {step}: parameters bit-equal to torch.optim.Adam (foreach) {eq}/{tot} = {eq / tot:.6f}")


@pytest.mark.parametrize('momentum,wd', [(0.9, 1e-4), (0.0, 0.0)])
@pytest.mark.parametrize('step', [1, 2, 1000])
def test_sgd_update_arithmetic(step, momentum, wd):
    ps = _params(7 + step)
    tp = _clone_params(ps)
    groups = lambda q: [{'params': q[:6]}, {'params': q[6:], 'lr': 0.003}]
    ours = optim.SGD(groups(ps), lr=0.01, momentum=momentum, weight_decay=wd)
    theirs = torch.optim.SGD(groups(tp), lr=0.01, momentum=momentum, weight_decay=wd, foreach=True)
    g = torch.Generator().manual_seed(200 + step)
    if step > 1 and momentum:
        for p, q in zip(ps, tp):
            b = torch.randn(p.shape, generator=g).to(DEV) * 1e-2
            ours.state[p] = {'momentum_buffer': b.clone()}
            theirs.state[q] = {'momentum_buffer': b.clone()}
    before = [(p.detach().cpu().numpy().copy(), p.grad.cpu().numpy().copy(),
               ours.state[p]['momentum_buffer'].cpu().numpy().copy() if (step > 1 and momentum) else None) for p in ps]
    ours.step()
    theirs.step()
    torch.cuda.synchronize()
    eq = tot = 0
    for i, (p, q) in enumerate(zip(ps, tp)):
        lr = ours.param_groups[0 if i < 6 else 1]['lr']
        p0, g0, b0 = before[i]
        first = b0 is None
        buf = (np.zeros(p.shape, np.float32) if first else b0) if momentum else None
        rp, rb = R.sgd(p0, g0, buf, -lr, wd, momentum, first)
        p64, bound = R.sgd_bound(p0, g0, buf, -lr, wd, momentum, first)
        e, n = _check(f"param {i}", p, rp, p64, bound, q)
        eq, tot = eq + e, tot + n
        if momentum:
            assert np.array_equal(_bits(ours.state[p]['momentum_buffer']), _canon(rb))
        else:
            assert 'momentum_buffer' not in ours.state[p]
    print(f"SGD(momentum {momentum}, wd {wd}) step {step}: bit-equal to torch.optim.SGD (foreach) {eq}/{tot} = {eq / tot:.6f}")


# ---------------------------------------------------------------------------------------------------------------------------
def _scene(name='config1_50k', seed=0):
    c = torch.from_numpy(synth.scene(name, seed=seed)).to(DEV)
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    return c, f


def _fresh_packs(eng):
    """what a newly built engine would pack from the current weights, per pack address"""
    convs = [(c0, False) for (c0, _) in eng.enc] + [(c0, eng.dense_up) for (c0, _) in eng.dec]
    convs += [(cv, False) for (_, blocks) in eng.enc + eng.dec for blk in blocks for cv in blk if cv is not None]
    convs.append((eng.final, False))
    out = {}
    for cv, wide in convs:
        w3 = cv.mod.kernel.detach()
        w3 = w3.unsqueeze(0) if w3.dim() == 2 else w3
        if cv.wpack is not None:
            out[cv.wpack.data_ptr()] = tc.pack_weights(w3.permute(1, 0, 2).reshape(1, cv.cin, cv.K * cv.cout) if wide else w3)
        if isinstance(cv.bwd, list):
            for (lo, hi, pk) in cv.bwd:
                out[pk.data_ptr()] = tc.pack_weights(w3[:, lo:hi, :], transpose_w=True)
    return out


def _grads(model):
    return [p.grad.detach().clone() for p in model.parameters()]


@pytest.mark.parametrize('arch,out', [('MinkUNet18A', 768), ('MinkUNet34C', 768), ('MinkUNet14A', 512)])
def test_step_repacks_in_place_and_the_next_step_equals_a_fresh_engine(arch, out, monkeypatch):
    c, f = _scene()
    mask = (torch.rand(len(c), generator=torch.Generator().manual_seed(3)) < 0.2).to(DEV)
    model = synth.randomize_bn_stats(synth.build_model(arch, out, seed=3), seed=7).train().to(DEV)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = optim.Adam(model.parameters(), lr=1e-3)
    opt.bind(eng)
    calls = []
    real = engine.FusedMinkUNet.refresh
    monkeypatch.setattr(engine.FusedMinkUNet, 'refresh', lambda self: (calls.append(1), real(self))[1])
    eng.forward_train(c, f, rows=mask).square().mean().backward()
    packs = {pk.data_ptr(): pk for (_, pk, *_r) in eng.repack_jobs()}
    versions = [p._version for p in model.parameters()]
    opt.step()
    assert all(p._version > v for p, v in zip(model.parameters(), versions))
    assert {pk.data_ptr() for (_, pk, *_r) in eng.repack_jobs()} == set(packs), "a pack moved"
    fresh = _fresh_packs(eng)
    assert set(fresh) == set(packs)
    for a, pk in packs.items():
        assert torch.equal(pk, fresh[a]), "a re-packed operand differs from a fresh pack of the updated weights"
    opt.zero_grad()
    y = eng.forward_train(c, f, rows=mask)
    y.square().mean().backward()
    g_bound = _grads(model)
    assert calls == []
    model.zero_grad()
    eng2 = engine.FusedMinkUNet(model, batch_stats=True)
    y2 = eng2.forward_train(c, f, rows=mask)
    y2.square().mean().backward()
    assert torch.equal(y, y2)
    assert all(torch.equal(a, b) for a, b in zip(g_bound, _grads(model)))


# ---------------------------------------------------------------------------------------------------------------------------
def _labels(coords, k):
    c64 = coords.long()
    lab = ((c64[:, 3] // 8) * 5 + c64[:, 1] // 16) % k
    lab[(c64[:, 1] * 7 + c64[:, 2] * 13 + c64[:, 3] * 3) % 10 == 0] = 255
    return lab


def _distill_run(model, make_opt, bind, steps=5):
    from openscene_b200 import distill
    c, f = _scene()
    g = torch.Generator().manual_seed(8)
    mask = (torch.rand(len(c), generator=g) < 0.2).to(DEV)
    tgt = torch.randn(int(mask.sum()), 768, generator=g).half().to(DEV)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = make_opt(model.parameters())
    if bind:
        opt.bind(eng)
    losses, after1 = [], None
    p0 = [p.detach().clone() for p in model.parameters()]
    for s in range(steps):
        opt.param_groups[0]['lr'] = 1e-3 * (1 - s / 100) ** 0.9
        torch.manual_seed(s)
        losses.append(float(distill.fused_distill_step(eng, opt, c, f, tgt, mask)))
        if s == 0:
            after1 = ([p.detach().clone() for p in model.parameters()], [p.grad.detach().clone() for p in model.parameters()])
    return losses, p0, after1, [p.detach().clone() for p in model.parameters()]


def _ce_run(model, make_opt, bind, steps=5):
    from openscene_b200 import train_mink
    coords = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=s, batch_index=s)) for s in range(2)])
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(2))
    c, f, lab = coords.to(DEV), feats.to(DEV), _labels(coords, 20).to(DEV)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = make_opt(model.parameters())
    if bind:
        opt.bind(eng)
    losses, after1 = [], None
    p0 = [p.detach().clone() for p in model.parameters()]
    for s in range(steps):
        torch.manual_seed(s)
        losses.append(float(train_mink.fused_train_step(eng, opt, c, f, lab)[0]))
        if s == 0:
            after1 = ([p.detach().clone() for p in model.parameters()], [p.grad.detach().clone() for p in model.parameters()])
    return losses, p0, after1, [p.detach().clone() for p in model.parameters()]


@pytest.mark.parametrize('kind', ['adam_distill', 'sgd_ce'])
def test_training_steps_match_torch_optim(kind):
    if kind == 'adam_distill':
        base = synth.randomize_bn_stats(synth.build_model('MinkUNet18A', 768, seed=3), seed=7).train()
        run, ours, theirs = _distill_run, (lambda ps: optim.Adam(ps, lr=1e-3)), (lambda ps: torch.optim.Adam(ps, lr=1e-3))
    else:
        base = synth.randomize_bn_stats(synth.build_model('MinkUNet18A', 20, seed=3), seed=7).train()
        kw = dict(lr=0.01, momentum=0.9, weight_decay=1e-4)
        run, ours, theirs = _ce_run, (lambda ps: optim.SGD(ps, **kw)), (lambda ps: torch.optim.SGD(ps, **kw))
    l_o, p0, (p1_o, g1), last_o = run(copy.deepcopy(base).to(DEV), ours, True)
    l_t, _, (p1_t, g1_t), _ = run(copy.deepcopy(base).to(DEV), theirs, False)
    l_o2, _, _, last_o2 = run(copy.deepcopy(base).to(DEV), ours, True)
    print(kind, 'losses ours', l_o, 'torch', l_t)
    for a, b in zip(l_o, l_t):
        assert abs(a - b) <= 1e-4 * abs(b)
    assert all(torch.equal(a, b) for a, b in zip(g1, g1_t)), "step 1 starts from the same gradients"
    eq = tot = 0
    for q0, g, a, b in zip(p0, g1, p1_o, p1_t):
        q0, g = q0.cpu().numpy(), g.cpu().numpy()
        if kind == 'adam_distill':
            lr = 1e-3
            p64, bound = R.adam_bound(q0, g, 0 * q0, 0 * q0, -(lr / (1 - 0.9)), (1 - 0.999) ** 0.5, 1 - 0.9, 0.999, 1 - 0.999,
                                      1e-8)
        else:
            p64, bound = R.sgd_bound(q0, g, 0 * q0, -0.01, 1e-4, 0.9, True)
        for x in (a, b):
            x = x.cpu().numpy().astype(np.float64)
            assert np.all(np.abs(x - p64) <= bound)
        eq += int((_bits(a) == _bits(b)).sum())
        tot += a.numel()
    print(f"{kind}: step-1 parameters bit-equal to torch.optim {eq}/{tot} = {eq / tot:.6f}")
    assert l_o == l_o2 and all(torch.equal(a, b) for a, b in zip(last_o, last_o2)), "two runs differ"


def test_checkpoints_interchange_with_torch_and_resume_exactly():
    from openscene_b200 import distill
    c, f = _scene()
    g = torch.Generator().manual_seed(8)
    mask = (torch.rand(len(c), generator=g) < 0.2).to(DEV)
    tgt = torch.randn(int(mask.sum()), 768, generator=g).half().to(DEV)
    base = synth.randomize_bn_stats(synth.build_model('MinkUNet14A', 768, seed=3), seed=7).train()

    def steps(model, opt, eng, k, first):
        for s in range(first, first + k):
            torch.manual_seed(s)
            distill.fused_distill_step(eng, opt, c, f, tgt, mask)

    def arm(model):
        eng = engine.FusedMinkUNet(model, batch_stats=True)
        opt = optim.Adam(model.parameters(), lr=1e-3)
        opt.bind(eng)
        return opt, eng

    m_a = copy.deepcopy(base).to(DEV)
    o_a, e_a = arm(m_a)
    steps(m_a, o_a, e_a, 3, 0)
    m_b = copy.deepcopy(base).to(DEV)
    o_b, e_b = arm(m_b)
    steps(m_b, o_b, e_b, 1, 0)
    buf = io.BytesIO()
    torch.save({'state_dict': m_b.state_dict(), 'optimizer': o_b.state_dict()}, buf)
    buf.seek(0)
    ck = torch.load(buf, weights_only=True)
    # the layout torch's own optimiser writes
    m_t = copy.deepcopy(base).to(DEV)
    o_t = torch.optim.Adam(m_t.parameters(), lr=1e-3)
    for p in m_t.parameters():
        p.grad = torch.zeros_like(p)
    o_t.step()
    ref = o_t.state_dict()
    assert ck['optimizer']['param_groups'] == ref['param_groups']
    for i, st in ref['state'].items():
        mine = ck['optimizer']['state'][i]
        assert mine.keys() == st.keys()
        for k in st:
            assert (mine[k].dtype, mine[k].device, mine[k].shape) == (st[k].dtype, st[k].device, st[k].shape), k
    o_t.load_state_dict(ck['optimizer'])                    # ours into torch ...
    o_x = optim.Adam(m_t.parameters(), lr=1e-3)
    o_x.load_state_dict(o_t.state_dict())                   # ... and torch's into ours
    assert all(torch.equal(o_x.state[p]['exp_avg'], o_t.state[p]['exp_avg']) for p in m_t.parameters())
    # resume: new model, engine and optimiser from the checkpoint, two more steps == three uninterrupted ones
    m_c = copy.deepcopy(base).to(DEV)
    m_c.load_state_dict(ck['state_dict'])
    o_c, e_c = arm(m_c)
    o_c.load_state_dict(ck['optimizer'])
    steps(m_c, o_c, e_c, 2, 1)
    for (n_, a), b in zip(m_a.named_parameters(), m_c.parameters()):
        assert torch.equal(a, b), n_
    for a, b in zip(m_a.buffers(), m_c.buffers()):
        assert torch.equal(a, b)


def test_other_consumers_see_the_step():
    import MinkowskiEngine as ME
    from openscene_b200 import fast_eval
    c, f = _scene()
    mask = (torch.rand(len(c), generator=torch.Generator().manual_seed(3)) < 0.2).to(DEV)
    model = synth.randomize_bn_stats(synth.build_model('MinkUNet18A', 768, seed=3), seed=7).to(DEV).eval()
    ev = engine.FusedMinkUNet(model)
    ff = fast_eval.install(model)

    def module_path(m):
        fast_eval.set_enabled(False)
        try:
            return m(ME.SparseTensor(f, c))
        finally:
            fast_eval.set_enabled(True)
    try:
        with torch.no_grad():
            ev(c, f)
            model(ME.SparseTensor(f, c))                     # fast_eval validates ...
            model(ME.SparseTensor(f, c))                     # ... and serves
            module_path(model)                               # the module path's pack cache holds the old weights
        assert ff.validated and ff.calls_fast == 1
        model.train()
        eng = engine.FusedMinkUNet(model, batch_stats=True)
        opt = optim.Adam(model.parameters(), lr=1e-2)
        opt.bind(eng)
        eng.forward_train(c, f, rows=mask).square().mean().backward()
        versions = [p._version for p in model.parameters()]
        opt.step()
        assert all(p._version > v for p, v in zip(model.parameters(), versions))
        model.eval()
        with torch.no_grad():
            out_new = engine.FusedMinkUNet(model)(c, f)
            assert torch.equal(ev(c, f), out_new), "the eval engine used stale packs"
            model(ME.SparseTensor(f, c))                     # re-validation after the weights changed ...
            t = model(ME.SparseTensor(f, c))                 # ... then the fast path again
            assert ff.validated and ff.calls_fast == 2
            assert torch.equal(t, out_new), "fast_eval used stale packs"
            a = module_path(model)
    finally:
        fast_eval.uninstall(model)
    fresh = copy.deepcopy(model)
    with torch.no_grad():
        assert torch.equal(a, module_path(fresh)), "the module path used a stale cached pack"


@pytest.mark.parametrize('arch', ['MinkUNet14A', 'MinkUNet34C'])
def test_bound_step_costs_two_library_launches(arch):
    c, f = _scene()
    model = synth.build_model(arch, 768, seed=3).train().to(DEV)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = optim.Adam(model.parameters(), lr=1e-3)
    eng.forward_train(c, f).square().mean().backward()
    n0 = C.lib().osb_launch_count()
    opt.step()
    assert C.lib().osb_launch_count() - n0 == 1
    opt.bind(eng)
    opt.zero_grad()
    eng.forward_train(c, f).square().mean().backward()
    n0 = C.lib().osb_launch_count()
    opt.step()
    assert C.lib().osb_launch_count() - n0 == 2
    print(arch, sum(p.numel() for p in model.parameters()), 'parameters: 2 launches per bound step')


def test_refusals_launch_nothing():
    def p_(x):
        p = torch.nn.Parameter(x)
        p.grad = torch.zeros_like(x)
        return p
    n0 = C.lib().osb_launch_count()
    for bad in ([p_(torch.randn(8, device=DEV).half())], [p_(torch.randn(8))], [p_(torch.randn(8, 2, device=DEV).t())],
                [p_(torch.randn(8, device=DEV)), p_(torch.randn(8))]):
        for opt in (optim.Adam(bad), optim.SGD(bad, lr=0.1, momentum=0.9)):
            with pytest.raises(NotImplementedError):
                opt.step()
            assert all(len(opt.state[p]) == 0 for p in bad)
    q = torch.nn.Parameter(torch.randn(4, 4, device=DEV))
    q.grad = torch.randn(4, 4, device=DEV).to_sparse()
    with pytest.raises(NotImplementedError, match='sparse'):
        optim.SGD([q], lr=0.1).step()
    for kw in (dict(amsgrad=True), dict(weight_decay=1e-4), dict(maximize=True), dict(fused=True)):
        with pytest.raises(NotImplementedError):
            optim.Adam([q], **kw)
    assert C.lib().osb_launch_count() == n0
    model = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV)
    ev = engine.FusedMinkUNet(model.eval())
    n0 = C.lib().osb_launch_count()
    with pytest.raises(ValueError, match='batch_stats'):
        optim.Adam(model.parameters()).bind(ev)
    assert C.lib().osb_launch_count() == n0
