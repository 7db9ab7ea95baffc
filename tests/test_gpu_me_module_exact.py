"""The MinkowskiEngine surface (openscene_b200/me.py) against the fp64 oracle ``oracle.me_cpu``, bit for bit.

Operands are dyadic (features {0, +-1, +-2} 2^-3, kernels, biases and output gradients {0, +-1, +-2, +-3} 2^-4, thinned where
the sums would grow), so every product is a multiple of the grid `g` of its two operands.  For each launch the test computes
the budget log2(max sum |terms| / g) from the oracle's own intermediate values and asserts it below 24 before comparing:
under it an fp32 accumulation is exact in any order, and the oracle's fp64 arithmetic is exact too, so the forward output,
``x.grad``, ``kernel.grad`` and ``bias.grad`` must be equal.  Both module routes run: ``OSB_MODULE_TC=1`` (the tensor-core
convolution for 32-multiple channels and K <= 32, bf16x3 split operands: exact only when every input and output gradient
is ``hi + lo`` exactly and every weight is bf16-exact, which the test asserts) and ``OSB_MODULE_TC=0`` (the CUDA-core
kernels everywhere).  Rows at coarse tensor strides are aligned with the oracle's by coordinates."""
import copy
import types

import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests import replay_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(params=['tc', 'cuda_core'])
def route(request, monkeypatch):
    monkeypatch.setenv('OSB_MODULE_TC', '1' if request.param == 'tc' else '0')
    return request.param


# ------------------------------------------------------------------ helpers
def _grid(t):
    """the largest power of two every entry of t is a multiple of"""
    v = t.detach().double().reshape(-1).cpu()
    v = v[v != 0]
    if not v.numel():
        return 1.0
    m, e = torch.frexp(v)
    mi = (m.abs() * 2.0 ** 53).long()
    low = (mi & -mi).double().log2()
    return float(torch.exp2((e.double() - 53 + low).min()))


def _hi_lo_exact(t):
    t = t.detach().float()
    hi = t.bfloat16().float()
    return torch.equal(hi + (t - hi).bfloat16().float(), t)


def _bf16_exact(t):
    return torch.equal(t.detach().float().bfloat16().float(), t.detach().float())


def _order(cg, co):
    """(og, oo) with cg[og] == co[oo] (integer coordinate rows)"""
    key = lambda a: (a[:, 0].astype(np.int64) << 60) + ((a[:, 1].astype(np.int64) + 4096) << 40) + \
        ((a[:, 2].astype(np.int64) + 4096) << 20) + (a[:, 3].astype(np.int64) + 4096)
    og, oo = np.argsort(key(cg)), np.argsort(key(co))
    assert np.array_equal(cg[og], co[oo])
    return torch.from_numpy(og), torch.from_numpy(oo)


def _thin(t, p, g):
    return t * (torch.rand(t.shape, generator=g) < p)


def _weights(shape, density, g):
    return _thin(R.probe_w(shape, g), density, g)


def _pair_managers(c, levels):
    from openscene_b200.coords import CoordinateManager
    from oracle import me_cpu
    om, cm = me_cpu.CoordinateManager(c), CoordinateManager(torch.from_numpy(c).to(DEV))
    ts = 1
    for _ in range(levels):
        om.stride(ts, 2), cm.stride(ts, 2)
        ts *= 2
    return om, cm


def _rows(cm, om, ts):
    """(og, oo): GPU rows og of the set at ts are the oracle's rows oo"""
    if ts == 1:
        n = len(om.coords[1])
        return torch.arange(n), torch.arange(n)
    return _order(cm.coords_external(ts).cpu().numpy(), om.coords[ts])


def _leaf(f, om, cm, ts):
    """the same leaf features on both sides (oracle row order in, GPU order made by coordinates)"""
    from openscene_b200 import me
    from oracle import me_cpu
    fo = f.double().clone().requires_grad_(True)
    og, oo = _rows(cm, om, ts)
    fg = torch.empty_like(f)
    fg[og] = f[oo]
    fg = fg.to(DEV).requires_grad_(True)
    return (fo, me_cpu.SparseTensor(fo, coordinate_manager=om, tensor_stride=ts),
            fg, me.SparseTensor(fg, coordinate_manager=cm, tensor_stride=ts), (og, oo))


def _out_rows(yg, yo, cm, om):
    return _rows(cm, om, yo.tensor_stride)


def _budget_layer(mo, xo, gout, what):
    """budgets (bits) of forward, dgrad and wgrad of oracle module mo on input SparseTensor xo with output gradient gout:
    A from the module on |x|, |W| (and autograd through it for sum |g||W| and sum |x||g|), g from the operands' grids"""
    from oracle import me_cpu
    ma = copy.deepcopy(mo)
    ma.kernel.data, ma.kernel.grad = mo.kernel.data.abs(), None
    if ma.bias is not None:
        ma.bias.data, ma.bias.grad = mo.bias.data.abs(), None
    fa = xo.F.detach().abs().clone().requires_grad_(True)
    ya = ma(me_cpu.SparseTensor(fa, coordinate_manager=xo.coordinate_manager, tensor_stride=xo.tensor_stride))
    (ya.F * gout.abs()).sum().backward()
    gx, gw, gg = _grid(xo.F), _grid(mo.kernel), _grid(gout)
    gf = gx * gw if mo.bias is None else min(gx * gw, _grid(mo.bias))
    bits = {'fwd': R.exact_budget_bits(ya.F.detach(), gf), 'dgrad': R.exact_budget_bits(fa.grad, gg * gw),
            'wgrad': R.exact_budget_bits(ma.kernel.grad, gx * gg)}
    for k, b in bits.items():
        assert b < 24, (what, k, b)
    return max(bits.values())


def _eq(a, b, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not torch.equal(a, b):
        d = (a - b).abs()
        raise AssertionError(f"{what}: {int((d > 0).sum())} of {d.numel()} entries differ, max |diff| {float(d.max()):.6g}")


def _modules(cls_o, cls_g, cin, cout, ks, stride, dil, bias, density, g):
    mo = cls_o(cin, cout, kernel_size=ks, stride=stride, dilation=dil, bias=bias, dimension=3).double()
    mg = cls_g(cin, cout, kernel_size=ks, stride=stride, dilation=dil, bias=bias, dimension=3)
    with torch.no_grad():
        mo.kernel.copy_(_weights(tuple(mo.kernel.shape), density, g).double())
        if bias:
            mo.bias.copy_(R.probe_w((1, cout), g).double())
    mg.load_state_dict({k: v.float() for k, v in mo.state_dict().items()})
    return mo, mg.to(DEV)


# ------------------------------------------------------------------ single layers
_CH = [(32, 64), (64, 32), (3, 32), (17, 45), (96, 20)]
_KS = [(1, 1, 1), (2, 2, 1), (3, 1, 1), (3, 2, 1), (3, 1, 2), (5, 1, 1)]
CONV_CASES = [(ks, st, dil, ci, co, i % 2 == 0, 1) for i, ((ks, st, dil), (ci, co)) in
              enumerate((a, b) for a in _KS for b in _CH)]
CONV_CASES += [(3, 1, 1, 32, 32, True, 2), (3, 2, 1, 17, 45, False, 2), (2, 2, 1, 64, 96, True, 2)]    # coarse-level inputs


def _layer(route, transpose, ks, stride, dil, cin, cout, bias, ts_in, seed=0):
    from openscene_b200 import me
    from oracle import me_cpu
    c = synth.random_cloud(2500, 24, seed=3, batch=2)
    g = torch.Generator().manual_seed(seed * 7919 + ks * 131 + cin * 17 + cout)
    levels = max(ts_in.bit_length() - 1 + (stride > 1 and not transpose), 1)
    om, cm = _pair_managers(c, levels)
    n_in = len(om.coords[ts_in])
    f = _thin(R.probe_x((n_in, cin), g), 0.75, g)
    K = ks ** 3
    density = min(1.0, 96.0 / (K * cin))
    cls = (me_cpu.MinkowskiConvolutionTranspose, me.MinkowskiConvolutionTranspose) if transpose else \
        (me_cpu.MinkowskiConvolution, me.MinkowskiConvolution)
    mo, mg = _modules(*cls, cin, cout, ks, stride, dil, bias, density, g)
    fo, xo, fg, xg, (ig, io) = _leaf(f, om, cm, ts_in)
    yo, yg = mo(xo), mg(xg)
    og, oo = _out_rows(yg, yo, cm, om)
    gout = R.probe_w(tuple(yo.F.shape), g).double()
    bits = _budget_layer(mo, xo, gout, (ks, stride, dil, cin, cout))
    tc_layer = route == 'tc' and cin % 32 == 0 and cout % 32 == 0 and (1 if mg.use_mm else K) <= 32
    if tc_layer:
        assert _hi_lo_exact(f) and _hi_lo_exact(gout) and _bf16_exact(mo.kernel)
    _eq(yg.F[og.to(DEV)], yo.F[oo], 'forward')
    gg = torch.empty(tuple(yo.F.shape), dtype=torch.float32)
    gg[og] = gout[oo].float()
    (yo.F * gout).sum().backward()
    (yg.F * gg.to(DEV)).sum().backward()
    _eq(fg.grad[ig.to(DEV)], fo.grad[io], 'x.grad')
    _eq(mg.kernel.grad, mo.kernel.grad, 'kernel.grad')
    if bias:
        _eq(mg.bias.grad, mo.bias.grad, 'bias.grad')
    return bits


@pytest.mark.parametrize('ks,stride,dil,cin,cout,bias,ts_in', CONV_CASES)
def test_convolution_exact(route, ks, stride, dil, cin, cout, bias, ts_in):
    _layer(route, False, ks, stride, dil, cin, cout, bias, ts_in)


@pytest.mark.parametrize('ks,cin,cout,bias', [(2, 64, 32, True), (2, 17, 45, False), (3, 32, 64, False), (3, 20, 17, True)])
def test_transposed_convolution_exact(route, ks, cin, cout, bias):
    """coarse leaf at tensor stride 2 -> stride 1; the backward runs on the transpose of the transposed map"""
    _layer(route, True, ks, 2, 1, cin, cout, bias, 2)


# ------------------------------------------------------------------ a short U-Net chain
def test_chain_stem_down_up_cat_head_exact(route):
    from openscene_b200 import me
    from oracle import me_cpu
    c = synth.random_cloud(1500, 20, seed=8, batch=2)
    g = torch.Generator().manual_seed(11)
    om, cm = _pair_managers(c, 1)
    n = len(c)
    f = _thin(R.probe_x((n, 3), g), 0.75, g)
    specs = [('stem', me_cpu.MinkowskiConvolution, me.MinkowskiConvolution, 3, 32, 5, 1, False, 0.25),
             ('down', me_cpu.MinkowskiConvolution, me.MinkowskiConvolution, 32, 64, 2, 2, True, 0.125),
             ('up', me_cpu.MinkowskiConvolutionTranspose, me.MinkowskiConvolutionTranspose, 64, 32, 2, 2, False, 0.125),
             ('head', me_cpu.MinkowskiConvolution, me.MinkowskiConvolution, 64, 20, 1, 1, True, 0.25)]
    mods = {name: _modules(co, cg, ci, cou, ks, st, 1, b, d, g) for (name, co, cg, ci, cou, ks, st, b, d) in specs}
    fo, xo, fg, xg, _ = _leaf(f, om, cm, 1)

    def run(x, side, M):
        s = M['stem'][side](x)
        d = M['down'][side](s)
        u = M['up'][side](d)
        cat = (me_cpu if side == 0 else me).cat(u, s)
        return M['head'][side](cat), (s, d, u, cat)

    yo, (so, do, uo, co) = run(xo, 0, mods)
    for t in (so, do, uo, co):
        t.F.retain_grad()
    yg, _ = run(xg, 1, mods)
    gout = _thin(R.probe_w((n, 20), g), 0.5, g).double()
    (yo.F * gout).sum().backward()
    (yg.F * gout.float().to(DEV)).sum().backward()
    # the budget of every layer, from the oracle's exact intermediate values and gradients
    bits = []
    for (name, *_), x, gy in zip(specs, (xo, so, do, co), (so.F.grad, do.F.grad, uo.F.grad, yo.F.grad)):
        gy = gout if name == 'head' else gy
        bits.append(_budget_layer(mods[name][0], x, gy, name))
        if route == 'tc' and name in ('down', 'up'):                  # the tensor-core layers: split operands must be exact
            assert _hi_lo_exact(x.F) and _hi_lo_exact(gy) and _bf16_exact(mods[name][0].kernel), name
    _eq(yg.F, yo.F, 'head output')
    _eq(fg.grad, fo.grad, 'x.grad')
    for name, (mo, mg) in mods.items():
        _eq(mg.kernel.grad, mo.kernel.grad, name + '.kernel.grad')
        if mo.bias is not None:
            _eq(mg.bias.grad, mo.bias.grad, name + '.bias.grad')
    print('chain budgets (bits):', ['%.1f' % b for b in bits])


# ------------------------------------------------------------------ pooling
@pytest.mark.parametrize('kind,c,ks,stride', [('sum', 20, 2, 2), ('sum', 32, 2, 2), ('sum', 32, 3, 1), ('avg', 20, 2, 2)])
def test_pooling_exact(route, kind, c, ks, stride):
    """sum pooling against the oracle; average pooling against the fp32 division of the exact sum by the count (the fp64
    oracle's quotient would be rounded twice), and its backward against the sum's backward of fp32(g / count)"""
    from openscene_b200 import me
    from oracle import me_cpu
    cl = synth.random_cloud(2500, 24, seed=5, batch=2)
    g = torch.Generator().manual_seed(c + ks)
    om, cm = _pair_managers(cl, 1)
    f = R.probe_x((len(cl), c), g)
    fo, xo, fg, xg, _ = _leaf(f, om, cm, 1)
    so = me_cpu.MinkowskiSumPooling(kernel_size=ks, stride=stride, dimension=3)(xo)
    pg = (me.MinkowskiSumPooling if kind == 'sum' else me.MinkowskiAvgPooling)(kernel_size=ks, stride=stride, dimension=3)
    yg = pg(xg)
    og, oo = _out_rows(yg, so, cm, om)
    gout = R.probe_w(tuple(so.F.shape), g).double()
    gg = torch.empty(tuple(so.F.shape), dtype=torch.float32)
    gg[og] = gout[oo].float()
    if kind == 'sum':
        ref, gref = so.F, gout
    else:
        ts_out = so.tensor_stride
        cnt = torch.zeros(len(om.coords[ts_out]), 1, dtype=torch.float64)
        for ii, oo_k in om.kernel_map(1, ts_out, ks):
            cnt.index_add_(0, oo_k, torch.ones(len(oo_k), 1, dtype=torch.float64))
        ref = (so.F.detach().float() / cnt.clamp(min=1).float()).double()
        gref = (gout.float() / cnt.clamp(min=1).float()).double()
    assert R.exact_budget_bits(so.F.detach().abs(), _grid(f)) < 24
    _eq(yg.F[og.to(DEV)], ref[oo], 'forward')
    (so.F * gref).sum().backward()
    (yg.F * gg.to(DEV)).sum().backward()
    _eq(fg.grad, fo.grad, 'x.grad')


# ------------------------------------------------------------------ at scale: the stem of distill_step
def test_stem_forward_and_weight_gradient_at_200k_exact():
    """MinkUNet's 5^3 stem (3 -> 32) on the 197k-voxel config2_200k scene in train mode, as distill_step runs it: the thin
    CUDA-core forward and weight gradient against fp64 on an independent neighbour search"""
    from openscene_b200 import me
    coords = torch.from_numpy(synth.scene('config2_200k')).to(DEV)
    n = coords.shape[0]
    g = torch.Generator(device=DEV).manual_seed(12)
    f = R.probe_x((n, 3), g, DEV)
    conv = me.MinkowskiConvolution(3, 32, kernel_size=5, dimension=3).to(DEV)
    with torch.no_grad():
        conv.kernel.copy_(R.probe_w((125, 3, 32), g, DEV))
    y = conv(me.SparseTensor(f, coords))
    gout = R.probe_w((n, 32), g, DEV)
    (y.F * gout).sum().backward()
    nbr = R.neighbour_map(coords, 5, 1)
    ref, A = R.conv(f.double(), nbr, n, conv.kernel.detach().double())
    assert R.exact_budget_bits(A, R.PROBE_GRID) < 24
    _eq(y.F, ref, 'stem forward')
    gw, Aw = R.wgrad(f.double(), nbr, gout.double(), 125)
    assert R.exact_budget_bits(Aw, R.PROBE_GRID) < 24
    _eq(conv.kernel.grad, gw, 'stem kernel.grad')


# ------------------------------------------------------------------ dtype refusals
def test_fp64_operands_are_refused():
    """a .double() module reaching the fp32 kernels raised nothing and read its fp64 weights as fp32 values"""
    from openscene_b200 import me
    c = torch.from_numpy(synth.random_cloud(500, 12, seed=1)).to(DEV)
    x = me.SparseTensor(torch.rand(len(c), 3, device=DEV), c)
    for ci, co, ks in ((3, 32, 5), (3, 20, 3)):
        conv = me.MinkowskiConvolution(ci, co, kernel_size=ks, dimension=3).to(DEV).double()
        with pytest.raises(TypeError, match='float64'):
            conv(x)
    cm = x.coordinate_manager
    with pytest.raises(TypeError, match='float64'):
        me.SparseTensor._wrap(torch.rand(len(c), 5, device=DEV, dtype=torch.float64), cm, 1).F


def test_fp16_operands_are_refused_before_any_launch(monkeypatch):
    """fp16 rows read as fp32 would be read and written out of bounds: nothing may be launched"""
    from openscene_b200 import _cabi, me
    c = torch.from_numpy(synth.random_cloud(500, 12, seed=2)).to(DEV)
    x = me.SparseTensor(torch.rand(len(c), 3, device=DEV), c)
    cm = x.coordinate_manager
    km = cm.kernel_map(1, 1, 3)
    n = cm.sets[1].n
    conv = me.MinkowskiConvolution(3, 20, kernel_size=3, dimension=3).to(DEV)
    launched = []

    def recorder(name, *args):
        launched.append(name)
        raise AssertionError(f"{name} was launched on fp16 operands")

    monkeypatch.setattr(_cabi, 'call', recorder)
    half = torch.rand(n, 3, device=DEV).half()
    with pytest.raises(TypeError, match='float16'):
        conv(me.SparseTensor._wrap(half, cm, 1))                            # _conv_raw
    with pytest.raises(TypeError, match='float16'):
        me.SparseTensor._wrap(torch.rand(n, 20, device=DEV).half(), cm, 1).F  # _RowGather (MinkowskiLinear under autocast)
    w3 = torch.rand(27, 3, 20, device=DEV)
    for xs, gs in ((torch.rand(n, 3, device=DEV), torch.rand(n, 20, device=DEV).half()),
                   (half, torch.rand(n, 20, device=DEV))):                  # the osb_conv_wgrad_f32 call
        ctx = types.SimpleNamespace(saved_tensors=(xs, w3), kmap=km, tc=False, needs_input_grad=(False, True), n_in=n)
        with pytest.raises(TypeError, match='float16'):
            me.SparseConvFunction.backward(ctx, gs)
    assert launched == []
