"""Every pooling module of the MinkowskiEngine surface, forward and backward through autograd, against the NumPy restatement
(tests/pool_ref.py) on the maps of the CPU oracle (rows aligned by coordinates); and the ResNet mirror on the GPU: the eval
forward against the reference forward's fp64 logits (tests/golden/live_resnets.npz) within the U-Net's 1e-3 per-row
yardstick, one train-mode step against the fp64 oracle under tests/test_gpu_unet.py's perturbed-oracle yardstick."""
import copy

import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests import pool_ref as P
from tests.test_resnet_mirror import LOGIT_ARCHS, mirror, oracle_me, resnet_cloud
from tests.util import golden, rel_row_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _bits(a):
    a = np.array(a, np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7fc00000                                          # one pattern for every NaN
    return b


def _order(cg, co):
    key = lambda a: (a[:, 0].astype(np.int64) << 60) + ((a[:, 1].astype(np.int64) + 4096) << 40) + \
        ((a[:, 2].astype(np.int64) + 4096) << 20) + (a[:, 3].astype(np.int64) + 4096)
    og, oo = np.argsort(key(cg)), np.argsort(key(co))
    assert np.array_equal(cg[og], co[oo])
    return og, oo


@pytest.mark.parametrize('name,mode', [('MinkowskiSumPooling', P.SUM), ('MinkowskiAvgPooling', P.AVG),
                                       ('MinkowskiMaxPooling', P.MAX)])
@pytest.mark.parametrize('ks,stride,dil,c', [(2, 2, 1, 32), (3, 1, 1, 20), (3, 2, 1, 7), (3, 1, 2, 96), (1, 2, 1, 5)])
def test_local_pooling_modules(name, mode, ks, stride, dil, c):
    import MinkowskiEngine as ME
    from oracle import me_cpu
    cl = synth.random_cloud(2000, 20, seed=ks + 3 * stride, batch=2)
    cl[:, 1:] -= 7                                                       # negative coordinates
    rng = np.random.RandomState(c)
    x_np = (rng.randn(len(cl), c) * 3).astype(np.float32)
    x_np[rng.rand(len(cl), c) < 0.1] = 1.0                               # ties
    om = me_cpu.CoordinateManager(cl)
    ts_out = om.stride(1, stride) if stride > 1 else 1
    maps = om.kernel_map(1, ts_out, ks, dil)
    nbr = np.full((len(maps), len(om.coords[ts_out])), -1, np.int64)
    for k, (ii, oo) in enumerate(maps):
        nbr[k, oo.numpy()] = ii.numpy()
    out, cnt, win = P.pool_fwd(x_np, nbr, mode)
    g_np = rng.randn(*out.shape).astype(np.float32)
    gin = P.pool_bwd(g_np, nbr, mode, cnt, win, len(cl))

    f = torch.from_numpy(x_np).to(DEV).requires_grad_(True)
    x = ME.SparseTensor(f, torch.from_numpy(cl).to(DEV))
    y = getattr(ME, name)(kernel_size=ks, stride=stride, dilation=dil, dimension=3)(x)
    assert y.tensor_stride == [ts_out] * 3
    og, oo = _order(y.C.cpu().numpy(), om.coords[ts_out])
    assert np.array_equal(_bits(y.F.detach().cpu().numpy()[og]), _bits(out[oo]))
    gg = np.empty_like(g_np)
    gg[og] = g_np[oo]
    (y.F * torch.from_numpy(gg).to(DEV)).sum().backward()
    assert np.array_equal(_bits(f.grad.cpu().numpy()), _bits(gin))


@pytest.mark.parametrize('name,mode', [('MinkowskiGlobalSumPooling', P.SUM), ('MinkowskiGlobalAvgPooling', P.AVG),
                                       ('MinkowskiGlobalMaxPooling', P.MAX)])
@pytest.mark.parametrize('ts', [1, 4])
def test_global_pooling_modules(name, mode, ts):
    """dyadic features (exact fp64 partials); batch rows interleaved at tensor stride 1, batch 1 empty"""
    import MinkowskiEngine as ME
    cl = synth.random_cloud(1500, 24, seed=2, batch=3)
    cl[cl[:, 0] == 1, 0] = 3
    cl = cl[np.random.RandomState(0).permutation(len(cl))]
    rng = np.random.RandomState(ts)
    c = 19
    x_np = (rng.randint(-50, 51, size=(len(cl), c)) * 2.0 ** -6).astype(np.float32)
    f = torch.from_numpy(x_np).to(DEV).requires_grad_(True)
    x = ME.SparseTensor(f, torch.from_numpy(cl).to(DEV))
    if ts > 1:
        x = ME.MinkowskiAvgPooling(kernel_size=ts, stride=ts, dimension=3)(x)
    feats = x.F.detach().cpu().numpy()
    batch = x.C[:, 0].cpu().numpy()
    pool = getattr(ME, name)(dimension=3)
    y = pool(x)
    assert y.shape == (4, c)
    ref, cnt, arg = P.global_fwd_exact(feats, batch, 4, mode)
    assert np.array_equal(_bits(y.detach().cpu().numpy()), _bits(ref))
    cm = x.coordinate_manager
    assert cm.batch_index(x._ts)[1] == 4 and pool(x).shape == (4, c)        # the count is cached per coordinate set
    g_np = rng.randn(4, c).astype(np.float32)
    y.backward(torch.from_numpy(g_np).to(DEV))
    if ts == 1:
        assert np.array_equal(_bits(f.grad.cpu().numpy()), _bits(P.global_bwd(g_np, batch, mode, cnt, arg)))
    else:
        assert torch.isfinite(f.grad).all()


def test_pooling_refuses_other_dtypes_before_any_launch(monkeypatch):
    from openscene_b200 import _cabi, me
    c = torch.from_numpy(synth.random_cloud(400, 10, seed=1)).to(DEV)
    x = me.SparseTensor(torch.rand(len(c), 4, device=DEV), c)
    cm = x.coordinate_manager
    cm.kernel_map(1, 1, 3)
    cm.batch_index(1)
    monkeypatch.setattr(_cabi, 'call', lambda name, *a: (_ for _ in ()).throw(AssertionError(f'{name} launched')))
    for dt in (torch.float16, torch.float64):
        xh = me.SparseTensor._wrap(torch.rand(len(c), 4, device=DEV).to(dt), cm, 1)
        for mod in (me.MinkowskiSumPooling(3, dimension=3), me.MinkowskiMaxPooling(3, dimension=3)):
            with pytest.raises(TypeError, match=str(dt).split('.')[1]):
                mod(xh)
    with pytest.raises(NotImplementedError):
        me.MinkowskiMaxPooling(kernel_size=[2, 2, 3], dimension=3)
    with pytest.raises(NotImplementedError):
        me.MinkowskiAvgPooling(kernel_size=2, kernel_generator=object(), dimension=3)


def test_linear_accepts_dense_and_sparse():
    from openscene_b200 import me
    lin = me.MinkowskiLinear(6, 3).to(DEV)
    d = torch.randn(4, 6, device=DEV)
    assert torch.equal(lin(d), lin.linear(d))
    c = torch.from_numpy(synth.random_cloud(100, 8, seed=1)).to(DEV)
    s = lin(me.SparseTensor(torch.randn(len(c), 6, device=DEV), c))
    assert isinstance(s, me.SparseTensor) and s.F.shape == (len(c), 3)


# ------------------------------------------------------------------ ResNet mirror
TOL = 1e-3


@pytest.mark.parametrize('arch', LOGIT_ARCHS)
def test_resnet_eval_forward_matches_the_reference_logits(arch):
    import MinkowskiEngine as ME
    g = golden('live_resnets.npz')
    coords, feats = resnet_cloud()
    model = mirror(arch).to(DEV).eval()
    with torch.no_grad():
        x = ME.SparseTensor(feats.to(DEV), torch.from_numpy(coords).to(DEV))
        y = model(x)
        assert 192 in x.coordinate_manager.sets and x.coordinate_manager.sets[192].n > 2   # conv5's tensor-stride-192 set
    assert rel_row_err(y.cpu().numpy(), g['logits'][LOGIT_ARCHS.index(arch)]) < TOL


def test_resnet_train_step_matches_the_oracle():
    """train-mode BN, cross-entropy, backward and one SGD step; truth = the fp64 oracle, yardstick = the fp64 oracle with
    every kernel perturbed by 2^-16 relative noise (tests/test_gpu_unet.py)"""
    from openscene_b200 import me
    from oracle import me_cpu
    coords, feats = resnet_cloud()
    labels = torch.tensor([3, 11])
    mg = mirror('ResNet14').to(DEV).train()
    m64 = mirror('ResNet14', ME=oracle_me()).double().train()
    m64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in mirror('ResNet14').state_dict().items()})
    mpt = copy.deepcopy(m64)
    gen = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n_, p_ in mpt.named_parameters():
            if n_.endswith('kernel'):
                p_.mul_(1 + 2.0 ** -16 * torch.randn(p_.shape, generator=gen, dtype=torch.float64))
    ce = torch.nn.CrossEntropyLoss()
    l64 = ce(m64(me_cpu.SparseTensor(feats.double(), torch.from_numpy(coords))), labels)
    lpt = ce(mpt(me_cpu.SparseTensor(feats.double(), torch.from_numpy(coords))), labels)
    lg = ce(mg(me.SparseTensor(feats.to(DEV), torch.from_numpy(coords).to(DEV))), labels.to(DEV))
    assert abs(l64.item() - lg.item()) < max(1e-5, 8 * abs(l64.item() - lpt.item()))
    l64.backward(); lpt.backward(); lg.backward()
    for (n, p64), (_, ppt), (_, pg) in zip(m64.named_parameters(), mpt.named_parameters(), mg.named_parameters()):
        a = p64.grad.numpy()
        e_pert = np.abs(a - ppt.grad.numpy()).max()
        e_gpu = np.abs(a - pg.grad.cpu().numpy().astype(np.float64)).max()
        scale = np.abs(a).max()
        assert e_gpu <= 10 * e_pert + 1e-3 * scale, (n, e_gpu, e_pert, scale)
    before = [p.detach().clone() for p in mg.parameters()]
    torch.optim.SGD(mg.parameters(), lr=0.1).step()                      # the step moves every weight by -lr * its gradient
    for p0, (n, p) in zip(before, mg.named_parameters()):
        torch.testing.assert_close(p.detach(), p0 - 0.1 * p.grad, rtol=1e-6, atol=1e-8, msg=n)
