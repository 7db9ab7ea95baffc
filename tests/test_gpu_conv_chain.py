"""Persistent convolution chains (csrc/conv_chain.cu) against the fp64 oracle: every layer shape of the U-Net through a
one-layer chain on a grid of 148 CTAs requested (more than the SMs: the launcher clamps it to one CTA per SM) and of 3 CTAs
(every CTA walks many items -> sub-tile pairing, ring wrap-around, both consumer warpgroups), forced split-K with the in-kernel reduction, the dense transposed form, and a
BasicBlock chain (conv1 | downsample -> barrier -> conv2 + residual) in ONE launch.  Tolerance 1e-4 relative per row.
Each configuration runs in its own process so that a trapped kernel cannot poison the CUDA context."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import synth, tc
from openscene_b200.coords import CoordinateManager
from oracle import me_cpu
grid, fsplit = int(sys.argv[1]), int(sys.argv[2])
cases = eval(sys.argv[3])
tc.tuning_set('chain_grid', grid); tc.tuning_set('chain_force_split', fsplit)
dev = torch.device('cuda:0')
def order(cg, co):
    key = lambda a: (a[:, 0].astype(np.int64) << 60) + ((a[:, 1].astype(np.int64) + 4096) << 40) + ((a[:, 2].astype(np.int64) + 4096) << 20) + (a[:, 3].astype(np.int64) + 4096)
    og, oo = np.argsort(key(cg)), np.argsort(key(co))
    m = np.empty(len(cg), dtype=np.int64); m[og] = oo          # gpu row -> oracle row
    return m
for (cin0, cin1, cout, ks, stride, epi) in cases:
    c = synth.scene('tiny') if ks != 1 else synth.random_cloud(700, 16, seed=1)
    cm = CoordinateManager(torch.from_numpy(c).to(dev))
    om = me_cpu.CoordinateManager(c)
    g = torch.Generator().manual_seed(0)
    cin = cin0 + cin1
    ts_in, ts_out = 1, 1
    if stride == 2:
        cm.stride(1, 2); om.stride(1, 2); ts_out = 2
    transposed = stride in (-2, -3)           # -3: the dense form (coarse rows x [W_0 | ... | W_7], scatter to children)
    if transposed:
        cm.stride(1, 2); om.stride(1, 2); ts_in, ts_out = 2, 1
    n_in, n_out = cm.sets[ts_in].n, cm.sets[ts_out].n
    K = ks ** 3
    if ks == 1:
        km_nbr = None
    elif transposed:
        km_nbr = cm.kernel_map(1, 2, ks).transposed().nbr
    else:
        km_nbr = cm.kernel_map(ts_in, ts_out, ks).nbr
    x = torch.randn(n_in, cin, generator=g)
    w = torch.randn(K, cin, cout, generator=g) / np.sqrt(K * cin / 2)
    co_in, co_out = om.coords[ts_in], om.coords[ts_out]
    m_in = order(cm.sets[ts_in].coords.cpu().numpy(), co_in)
    m_out = order(cm.sets[ts_out].coords.cpu().numpy(), co_out)
    x_o = torch.zeros(n_in, cin, dtype=torch.float64); x_o[m_in] = x.double()
    if ks == 1:
        ref_o = x_o @ w[0].double()
    else:
        maps = om.kernel_map(1, 2, ks) if transposed else om.kernel_map(ts_in, ts_out, ks)
        if transposed: maps = [(oo, ii) for ii, oo in maps]
        ref_o = me_cpu._conv_apply(x_o, maps, w.double(), n_out)
    scale = shift = None
    res_f = None
    if 'bn' in epi:
        scale = (0.5 + torch.rand(cout, generator=g)); shift = torch.randn(cout, generator=g) * 0.1
        ref_o = ref_o * scale.double() + shift.double()
    if 'res' in epi:
        res_f = torch.randn(n_out, cout, generator=g)
        r_o = torch.zeros(n_out, cout, dtype=torch.float64); r_o[m_out] = res_f.double()
        ref_o = ref_o + r_o
    if 'relu' in epi:
        ref_o = torch.relu(ref_o)
    ref = ref_o[m_out]
    xd = x.to(dev)
    s0 = tc.to_split(xd[:, :cin0].contiguous())
    s1 = tc.to_split(xd[:, cin0:].contiguous()) if cin1 else None
    rs = tc.to_split(res_f.to(dev)) if res_f is not None else None
    sc = scale.to(dev) if scale is not None else None
    sh = shift.to(dev) if shift is not None else None
    if stride == -3:
        wide = w.permute(1, 0, 2).reshape(1, cin, K * cout).contiguous()
        wt = tc.pack_weight_tiles(wide.to(dev))
        down = cm.kernel_map(1, 2, ks).nbr                      # [K, n_coarse]: child row of parent o through offset k
        o_split, o_f32 = tc.conv_chain_single(s0, cin0, None, 0, None, n_in, 1, wt, K * cout, sc, sh, None, 'relu' in epi, True, True,
                                              None, cmap=down, cmap_cout=cout, n_rows_out=n_out)
    else:
        wt = tc.pack_weight_tiles(w.to(dev))
        o_split, o_f32 = tc.conv_chain_single(s0, cin0, s1, cin1, km_nbr, n_out, K, wt, cout, sc, sh, rs, 'relu' in epi, True, True, None)
    torch.cuda.synchronize()
    def err(a):
        a = a.double().cpu()
        return float(((a - ref).norm(dim=1) / (ref.norm(dim=1) + 1e-6)).max())
    e1, e2 = err(o_f32), err(tc.from_split(o_split, cout))
    print('RESULT grid', grid, 'split', fsplit, cin0, cin1, cout, ks, stride, epi, 'n_out', n_out, 'err_f32=%%.3e err_split=%%.3e' %% (e1, e2), flush=True)
    assert e1 < 1e-4 and e2 < 1e-4, (e1, e2)
    if stride != -3:                                            # scattered fp32 output == plain output permuted
        perm = torch.randperm(n_out, generator=g).to(dev).int()
        _, o_sc = tc.conv_chain_single(s0, cin0, s1, cin1, km_nbr, n_out, K, wt, cout, None, None, None, False, False, True, perm)
        _, o_pl = tc.conv_chain_single(s0, cin0, s1, cin1, km_nbr, n_out, K, wt, cout, None, None, None, False, False, True, None)
        assert torch.equal(o_sc[perm.long()], o_pl)
        # bit-identical to itself run to run (fixed-order reduction)
        _, o_pl2 = tc.conv_chain_single(s0, cin0, s1, cin1, km_nbr, n_out, K, wt, cout, None, None, None, False, False, True, None)
        assert torch.equal(o_pl2, o_pl)
print('OK')
'''

CASES = [
    # cin0 cin1 cout ks stride epilogue
    (32, 0, 32, 3, 1, 'none'), (96, 0, 96, 3, 1, 'bn+relu'), (96, 0, 96, 3, 1, 'bn+res+relu'), (128, 64, 128, 3, 1, 'bn+relu'),
    (32, 0, 32, 2, 2, 'bn+relu'), (256, 0, 128, 2, -2, 'bn+relu'), (96, 32, 96, 1, 1, 'bn'), (96, 0, 768, 1, 1, 'none'),
    (256, 128, 256, 3, 1, 'bn+relu'), (64, 0, 64, 3, 1, 'none'),
    (256, 0, 128, 2, -3, 'bn+relu'), (96, 0, 96, 2, -3, 'bn+relu'),
]


def _run(grid, fsplit, cases, timeout=420):
    src = WORKER % {'root': ROOT}
    r = subprocess.run([sys.executable, '-c', src, str(grid), str(fsplit), repr(cases)], capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


@pytest.mark.parametrize('grid', [148, 3])
def test_chain_single_layers(grid):
    _run(grid, 0, CASES)


@pytest.mark.parametrize('grid,fsplit', [(148, 4), (5, 3), (148, 32)])
def test_chain_forced_split(grid, fsplit):
    _run(grid, fsplit, [CASES[2], CASES[3], CASES[4], CASES[8], CASES[6]])


def test_chain_basic_block_in_one_launch():
    """conv1 (3^3, BN, ReLU) and the 1x1x1 downsample read x; a grid barrier; conv2 (3^3, BN) + residual + ReLU: one launch,
    with and without split-K, against the per-layer oracle."""
    src = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import synth, tc, _cabi as C
from openscene_b200.coords import CoordinateManager
from oracle import me_cpu
dev = torch.device('cuda:0')
c = synth.scene('tiny')
cm = CoordinateManager(torch.from_numpy(c).to(dev))
om = me_cpu.CoordinateManager(c)
n = cm.sets[1].n
nbr = cm.kernel_map(1, 1, 3).nbr
key = lambda a: (a[:, 0].astype(np.int64) << 60) + ((a[:, 1].astype(np.int64) + 4096) << 40) + ((a[:, 2].astype(np.int64) + 4096) << 20) + (a[:, 3].astype(np.int64) + 4096)
og, oo = np.argsort(key(cm.sets[1].coords.cpu().numpy())), np.argsort(key(om.coords[1]))
m = np.empty(n, dtype=np.int64); m[og] = oo
g = torch.Generator().manual_seed(1)
cin, cmid = 192, 128
x = torch.randn(n, cin, generator=g)
w1 = torch.randn(27, cin, cmid, generator=g) / np.sqrt(27 * cin / 2)
w2 = torch.randn(27, cmid, cmid, generator=g) / np.sqrt(27 * cmid / 2)
wd = torch.randn(1, cin, cmid, generator=g) / np.sqrt(cin / 2)
bn = lambda: (0.5 + torch.rand(cmid, generator=g), torch.randn(cmid, generator=g) * 0.1)
(s1, b1), (s2, b2), (sd, bd) = bn(), bn(), bn()
maps = om.kernel_map(1, 1, 3)
xo = torch.zeros(n, cin, dtype=torch.float64); xo[m] = x.double()
y = torch.relu(me_cpu._conv_apply(xo, maps, w1.double(), n) * s1.double() + b1.double())
r = (xo @ wd[0].double()) * sd.double() + bd.double()
ref = torch.relu(me_cpu._conv_apply(y, maps, w2.double(), n) * s2.double() + b2.double() + r)[m]
xs = tc.to_split(x.to(dev))
wt1, wt2, wtd = (tc.pack_weight_tiles(t.to(dev)) for t in (w1, w2, wd))
dv = lambda t: t.to(dev)
cs = [dv(t) for t in (s1, b1, s2, b2, sd, bd)]
for grid, fsplit in ((148, 0), (148, 6), (4, 0), (7, 2)):
    tc.tuning_set('chain_grid', grid); tc.tuning_set('chain_force_split', fsplit)
    y_s = torch.empty((n, 4 * cmid), dtype=torch.uint8, device=dev)
    r_s = torch.empty((n, 4 * cmid), dtype=torch.uint8, device=dev)
    o_s = torch.empty((n, 4 * cmid), dtype=torch.uint8, device=dev)
    wsb = [C.lib().osb_conv_chain_workspace_bytes(n, K, ci, cmid) for (K, ci) in ((27, cin), (1, cin), (27, cmid))]
    ws = [torch.empty(max(b, 16), dtype=torch.uint8, device=dev) for b in wsb]
    ch = tc.ConvChain(dev, 8)
    ch.add(xs.data_ptr(), cin, 0, 0, nbr.data_ptr(), n, 27, wt1.data_ptr(), cmid, cs[0].data_ptr(), cs[1].data_ptr(), 0, 1, y_s.data_ptr(),
           ws=ws[0].data_ptr(), ws_bytes=wsb[0])
    ch.add(xs.data_ptr(), cin, 0, 0, 0, n, 1, wtd.data_ptr(), cmid, cs[4].data_ptr(), cs[5].data_ptr(), 0, 0, r_s.data_ptr(),
           ws=ws[1].data_ptr(), ws_bytes=wsb[1])
    ch.add(y_s.data_ptr(), cmid, 0, 0, nbr.data_ptr(), n, 27, wt2.data_ptr(), cmid, cs[2].data_ptr(), cs[3].data_ptr(), r_s.data_ptr(), 1,
           o_s.data_ptr(), ws=ws[2].data_ptr(), ws_bytes=wsb[2], barrier_before=1)
    for rep in range(3):                      # the grid barrier words are reused launch after launch without a reset
        ch.run()
    torch.cuda.synchronize()
    out = tc.from_split(o_s, cmid).double().cpu()
    e = float(((out - ref).norm(dim=1) / (ref.norm(dim=1) + 1e-6)).max())
    print('RESULT block grid', grid, 'split', fsplit, 'err %%.3e' %% e, flush=True)
    assert e < 1e-4, e
print('OK')
''' % {'root': ROOT}
    r = subprocess.run([sys.executable, '-c', src], capture_output=True, text=True, timeout=420)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]
