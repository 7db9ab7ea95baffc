"""Train-mode BatchNorm on the device (csrc/bn_train.cu) and ``FusedMinkUNet(model, batch_stats=True)``: the forward
run/distill.py's validate() makes (train mode under no_grad), which normalises every layer with batch statistics and moves
the running buffers.

* the kernels through the C ABI against ``F.batch_norm(training=True)`` in fp64, with per-channel means up to 10^3 sigma;
* the engine against the module path (output and every BatchNorm's buffers over three consecutive calls), and against the
  fp64 oracle with the 2^-16-perturbed-oracle yardstick of tests/test_gpu_unet.py;
* determinism, the interplay with eval-mode engines / fast_eval (version bumps, no re-pack on its own updates), refusals."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from openscene_b200 import _cabi as C
from openscene_b200 import synth
from tests import norm_ref as NR
from tests.util import rel_row_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _to_split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _joined(rows, c):
    out = torch.empty((rows.shape[0], c), dtype=torch.float32, device=DEV)
    C.call('osb_split_to_f32', C.ptr(rows), rows.shape[0], c, C.ptr(out), C.stream_ptr())
    return out


def _rows(n, c, seed):
    """split rows whose channels have sigma in [e^-2, e^2] and means up to 10^3 sigma -> (rows, joined fp64, sigma)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    sigma = torch.exp(4 * torch.rand(c, device=DEV, generator=g) - 2)
    mean = sigma * (2000 * torch.rand(c, device=DEV, generator=g) - 1000)
    x = mean + sigma * torch.randn(n, c, device=DEV, generator=g)
    rows = _to_split(x)
    return rows, _joined(rows, c).double(), sigma.double()


class _BN:
    """the device buffers of one nn.BatchNorm1d plus the engine-side outputs"""

    def __init__(self, c, seed, nbt=5):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.w = 0.5 + torch.rand(c, device=DEV, generator=g)
        self.b = torch.rand(c, device=DEV, generator=g) - 0.5
        self.rm = torch.rand(c, device=DEV, generator=g) - 0.5
        self.rv = 0.5 + torch.rand(c, device=DEV, generator=g)
        self.nbt = torch.full((1,), nbt, dtype=torch.int64, device=DEV)
        self.scale = torch.empty(c, device=DEV)
        self.shift = torch.empty(c, device=DEV)

    def stats(self, rows, n, c, eps, momentum):
        ws_bytes = C.lib().osb_bn_stats_workspace_bytes(n, c)
        assert ws_bytes > 0
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
        C.call('osb_bn_batch_stats', rows.data_ptr(), n, c, self.w.data_ptr(), self.b.data_ptr(), eps,
               -1.0 if momentum is None else momentum, self.rm.data_ptr(), self.rv.data_ptr(), self.nbt.data_ptr(),
               self.scale.data_ptr(), self.shift.data_ptr(), ws.data_ptr(), ws_bytes, C.stream_ptr())

    def state(self):
        return [t.clone() for t in (self.rm, self.rv, self.nbt, self.scale, self.shift)]


def _apply(rows, n, c, bn, res=None, res_bn=None, relu=1):
    out = rows.clone()
    C.call('osb_bn_apply_split', out.data_ptr(), n, c, bn.scale.data_ptr(), bn.shift.data_ptr(),
           res.data_ptr() if res is not None else None, res_bn.scale.data_ptr() if res_bn else None,
           res_bn.shift.data_ptr() if res_bn else None, relu, C.stream_ptr())
    return out


@pytest.mark.parametrize('momentum', [0.1, None])
@pytest.mark.parametrize('c', [32, 96, 256])
@pytest.mark.parametrize('n', [2, 3, 129, 4099, 197383])
def test_kernels_match_torch_batch_norm(n, c, momentum):
    eps = 1e-5
    rows, x, sigma = _rows(n, c, seed=n * 7 + c)
    bn = _BN(c, seed=c)
    rm0, rv0, nbt0 = bn.rm.double(), bn.rv.double(), int(bn.nbt)
    bn.stats(rows, n, c, eps, momentum)
    # fp64 reference: torch's own train-mode BatchNorm on the joined values (the factor for momentum=None: 1 / tracked batches)
    m = 1.0 / (nbt0 + 1) if momentum is None else momentum
    rm_ref, rv_ref = rm0.clone(), rv0.clone()
    w64, b64 = bn.w.double(), bn.b.double()
    F.batch_norm(x, rm_ref, rv_ref, w64, b64, training=True, momentum=m, eps=eps)
    mean, var = x.mean(0), x.var(0, unbiased=False)
    scale_ref = w64 / torch.sqrt(var + eps)
    torch.cuda.synchronize()
    assert int(bn.nbt) == nbt0 + 1
    sc, sh = bn.scale.double(), bn.shift.double()
    # scale / shift and the running buffers (torch's update above, unbiased variance) per channel within the bounds of
    # tests/norm_ref.py: the fp64 sums' depth term carried through the finalize arithmetic, plus one fp32 rounding
    ref = NR.bn_stats(x, bn.w, bn.b, eps)
    bd = NR.stats_bounds(ref, rm0, rv0, m)
    for name, got, want in (('scale', sc, ref['scale']), ('shift', sh, ref['shift']), ('running_mean', bn.rm, rm_ref),
                            ('running_var', bn.rv, rv_ref)):
        assert bool(((got.double() - want).abs() <= bd[name]).all()), name
    assert torch.allclose(ref['scale'], scale_ref, rtol=1e-12) and torch.allclose(ref['mean'], mean, rtol=1e-12, atol=1e-12)
    # two runs: bit-identical statistics
    first = bn.state()
    bn.rm.copy_(rm0.float()); bn.rv.copy_(rv0.float()); bn.nbt.fill_(nbt0)
    bn.stats(rows, n, c, eps, momentum)
    assert all(torch.equal(a, b) for a, b in zip(first, bn.state()))

    if momentum is None:
        return
    # apply, in place on split rows: every residual form, ReLU on and off, against the fp64 statistics (so the hand-off
    # from the statistics launch is measured), with the per-element bound of tests/norm_ref.py
    res_rows, res_x, _ = _rows(n, c, seed=n * 7 + c + 1)
    res_bn = _BN(c, seed=c + 1)
    res_bn.stats(res_rows, n, c, eps, momentum)
    rref = NR.bn_stats(res_x, res_bn.w, res_bn.b, eps)
    for form in ('none', 'identity', 'normalised'):
        for relu in (0, 1):
            res = None if form == 'none' else res_rows
            out = _apply(rows, n, c, bn, res=res, res_bn=res_bn if form == 'normalised' else None, relu=relu)
            y_ref, tol = NR.bn_apply(x, ref, None if form == 'none' else res_x, rref if form == 'normalised' else None, bool(relu))
            got = _joined(out, c).double()
            assert bool(((got - y_ref).abs() <= tol).all()), (form, relu, float(((got - y_ref).abs() / tol).max()))
            out2 = _apply(rows, n, c, bn, res=res, res_bn=res_bn if form == 'normalised' else None, relu=relu)
            assert torch.equal(out, out2)
    # the residual rows are read, never written
    assert torch.equal(_joined(res_rows, c).double(), res_x)


# ---------------------------------------------------------------------------------------------------------------------------
def _bns(model):
    return [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)]


def _buffers_close(a, b, tol=1e-3):
    ba, bb = _bns(a), _bns(b)
    assert len(ba) == len(bb)
    for x, y in zip(ba, bb):
        for name in ('running_mean', 'running_var'):
            p, q = getattr(x, name), getattr(y, name)
            assert float((p - q).abs().max()) <= tol * float(q.abs().max()), name
        assert int(x.num_batches_tracked) == int(y.num_batches_tracked)


CASES = [('config1_50k', 'MinkUNet18A', 768, 48), ('config1_50k', 'MinkUNet34C', 768, 62),
         ('batch3', 'MinkUNet14A', 512, None), ('batch3', 'MinkUNet18B', 20, None)]


def _scene(name):
    c = synth.random_cloud(3000, 36, seed=4, batch=3) if name == 'batch3' else synth.scene(name)
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(2))
    return torch.from_numpy(c).to(DEV), f.to(DEV)


@pytest.mark.parametrize('momentum', [0.1, None])
@pytest.mark.parametrize('scene,arch,head,n_bn', CASES)
def test_engine_matches_module_path(scene, arch, head, n_bn, momentum):
    import MinkowskiEngine as ME
    from openscene_b200 import engine
    c, f = _scene(scene)
    model = synth.randomize_bn_stats(synth.build_model(arch, head, seed=3), seed=7).train()
    if momentum is None:
        for m in _bns(model):
            m.momentum = None
    if n_bn is not None:
        assert len(_bns(model)) == n_bn
    m_mod, m_eng = copy.deepcopy(model).to(DEV), copy.deepcopy(model).to(DEV)
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    for step in range(3):
        with torch.no_grad():
            ref = m_mod(ME.SparseTensor(f, c))
        out = eng(c, f)
        assert out.shape == ref.shape
        err = rel_row_err(out.cpu().numpy(), ref.cpu().numpy())
        print(scene, arch, head, momentum, 'step', step, 'rel err', err)
        assert err < 1e-3
        _buffers_close(m_eng, m_mod)


def test_engine_against_fp64_oracle():
    """Tiny scene, train-mode BatchNorm over the handful of voxels of the coarse levels (ill-conditioned): the yardstick is
    the fp64 oracle with every kernel perturbed by 2^-16 relative noise, as in tests/test_gpu_unet.py."""
    from openscene_b200 import engine
    from oracle import me_cpu
    c = synth.scene('tiny')
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(0))
    m64 = synth.build_model('MinkUNet14A', 64, seed=0, ME=me_cpu.as_module()).double().train()
    mpt = copy.deepcopy(m64)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n_, p_ in mpt.named_parameters():
            if n_.endswith('kernel'):
                p_.mul_(1 + 2.0 ** -16 * torch.randn(p_.shape, generator=g, dtype=torch.float64))
        o64 = m64(me_cpu.SparseTensor(f.double(), torch.from_numpy(c)))
        opt = mpt(me_cpu.SparseTensor(f.double(), torch.from_numpy(c)))
    mg = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV).train()
    og = engine.FusedMinkUNet(mg, batch_stats=True)(torch.from_numpy(c).to(DEV), f.to(DEV))
    e_fwd = rel_row_err(og.cpu().numpy(), o64.numpy())
    e_pert = rel_row_err(opt.numpy(), o64.numpy())
    print('forward rel err: engine', e_fwd, ' 2^-16-perturbed oracle', e_pert)
    assert e_fwd < max(1e-3, 8 * e_pert)
    assert torch.allclose(m64.bn0.bn.running_mean.float(), mg.bn0.bn.running_mean.cpu(), atol=1e-5)
    assert torch.allclose(m64.bn0.bn.running_var.float(), mg.bn0.bn.running_var.cpu(), atol=1e-5)
    assert int(mg.bn0.bn.num_batches_tracked) == int(m64.bn0.bn.num_batches_tracked) == 1


def test_engine_is_deterministic():
    from openscene_b200 import engine
    c, f = _scene('config1_50k')
    model = synth.build_model('MinkUNet34C', 768, seed=1).to(DEV).train()
    snap = {k: v.clone() for k, v in model.state_dict().items()}
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    o1 = eng(c, f).clone()
    b1 = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        for k, v in model.state_dict().items():
            v.copy_(snap[k])
    o2 = eng(c, f)
    assert torch.equal(o1, o2)
    assert all(torch.equal(b1[k], v) for k, v in model.state_dict().items())
    assert any(not torch.equal(b1[k], snap[k]) for k in snap if k.endswith('running_mean'))


def test_eval_engine_and_fast_eval_pick_up_moved_statistics(monkeypatch):
    import MinkowskiEngine as ME
    from openscene_b200 import engine, fast_eval
    assert fast_eval.enabled()
    c, f = _scene('config1_50k')
    model = synth.build_model('MinkUNet18A', 768, seed=2).to(DEV).eval()
    eng_eval = engine.FusedMinkUNet(model)
    out0 = eng_eval(c, f).clone()
    with torch.no_grad():                 # fast_eval: root found (module path), validated (both paths), then the engine serves
        for _ in range(3):
            model(ME.SparseTensor(f, c))
    ff = model._osb_fast
    assert ff.disabled is None and ff.validated and ff.calls_fast == 1
    model.train()
    builds = []
    orig = engine.FusedMinkUNet._build
    monkeypatch.setattr(engine.FusedMinkUNet, '_build', lambda self: (builds.append(self), orig(self))[1])
    eng_bs = engine.FusedMinkUNet(model, batch_stats=True)
    assert len(builds) == 1
    for _ in range(3):
        eng_bs(c, f)
    assert len(builds) == 1                                     # its own running-buffer updates cost no re-pack
    model.eval()
    # the eval-mode engine re-folds the moved statistics: equal to the eval module path with the new buffers
    out1 = eng_eval(c, f)
    assert len(builds) == 2 and builds[-1] is eng_eval
    with torch.no_grad():
        ref = ff.orig(ME.SparseTensor(f, c))                    # the module path itself, bypassing fast_eval
    assert rel_row_err(out1.cpu().numpy(), ref.cpu().numpy()) < 1e-3
    assert rel_row_err(out1.cpu().numpy(), out0.cpu().numpy()) > 1e-3
    # fast_eval re-validates: the next call runs both paths (no fast call), the one after is served by the engine again
    with torch.no_grad():
        v = model(ME.SparseTensor(f, c))
        assert ff.calls_fast == 1 and ff.validated
        w = model(ME.SparseTensor(f, c))
    assert ff.calls_fast == 2
    assert rel_row_err(v.cpu().numpy(), ref.cpu().numpy()) < 1e-6
    assert rel_row_err(w.cpu().numpy(), ref.cpu().numpy()) < 1e-3
    # a change of a BatchNorm weight or of a kernel is not missed by the batch-statistics engine
    model.train()
    n_builds = len(builds)
    m_mod = synth.build_model('MinkUNet18A', 768, seed=2)              # a copy without fast_eval's wrapper
    m_mod.load_state_dict(model.state_dict())
    m_mod = m_mod.to(DEV).train()
    for m in (model, m_mod):
        with torch.no_grad():
            m.block1[0].norm1.bn.weight.mul_(1.5)
            m.block3[0].conv2.kernel.add_(0.01)
    out = eng_bs(c, f)
    assert len(builds) == n_builds + 1
    with torch.no_grad():
        ref = m_mod(ME.SparseTensor(f, c))
    assert rel_row_err(out.cpu().numpy(), ref.cpu().numpy()) < 1e-3
    _buffers_close(model, m_mod)


def test_refusals():
    from openscene_b200 import engine
    model = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV)
    with pytest.raises(RuntimeError, match='train'):
        engine.FusedMinkUNet(model.eval(), batch_stats=True)
    with pytest.raises(RuntimeError, match='eval'):
        engine.FusedMinkUNet(model.train())
    for attr in ('affine', 'track_running_stats'):
        m = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV).train()
        bn = m.block1[0].norm1.bn
        setattr(bn, attr, False)
        if attr == 'affine':
            bn.weight = bn.bias = None
        else:
            bn.running_mean = bn.running_var = bn.num_batches_tracked = None
        with pytest.raises(NotImplementedError, match='BatchNorm'):
            engine.FusedMinkUNet(m, batch_stats=True)
    m = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV).train()
    m.bn0.bn.running_mean = m.bn0.bn.running_mean.double()
    with pytest.raises(NotImplementedError, match='fp32'):
        engine.FusedMinkUNet(m, batch_stats=True)
    eng = engine.FusedMinkUNet(model.train(), batch_stats=True)
    text = torch.nn.functional.normalize(torch.randn(4, 64, device=DEV), dim=1)
    with pytest.raises(NotImplementedError, match='eval-only'):
        eng.fold_head(text)
    # fewer than 2 rows at the coarsest level (every voxel inside one 16^3 cell): refused before any launch, no buffer moves
    c = torch.from_numpy(synth.random_cloud(300, 12, seed=1)).to(DEV)
    f = torch.ones(c.shape[0], 3, device=DEV)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    versions = [t._version for t in model.buffers()]
    with pytest.raises(ValueError, match='Expected more than 1 value per channel when training'):
        eng(c, f)
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    assert versions == [t._version for t in model.buffers()]
    # the module path refuses the same input (torch's own check, one level later than the engine)
    import MinkowskiEngine as ME
    with pytest.raises(ValueError, match='Expected more than 1 value per channel when training'), torch.no_grad():
        copy.deepcopy(model)(ME.SparseTensor(f, c))
