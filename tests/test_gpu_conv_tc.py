"""Tensor-core (wgmma) sparse convolution (csrc/conv_tc.cu) and the fused stem (csrc/conv_stem.cu)
against the fp64 oracle.  bf16x3 split arithmetic: tolerance 1e-4 relative per row (observed ~1e-5).
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
mode, cin0, cin1, cout, ks, stride, epi = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6]), sys.argv[7]
tc.debug_set_tc({'cpasync': 2, 'rows': 0}[mode], 0)
dev = torch.device('cuda:0')
c = synth.scene('tiny') if ks != 1 else synth.random_cloud(700, 16, seed=1)
cm = CoordinateManager(torch.from_numpy(c).to(dev))
om = me_cpu.CoordinateManager(c)
g = torch.Generator().manual_seed(0)
cin = cin0 + cin1
ts_in, ts_out = 1, 1
if stride == 2:
    cm.stride(1, 2); om.stride(1, 2); ts_out = 2
transposed = stride == -2
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
# oracle in fp64, rows aligned through coordinates
co_in, co_out = om.coords[ts_in], om.coords[ts_out]
def order(cg, co):
    key = lambda a: (a[:, 0].astype(np.int64) << 60) + ((a[:, 1].astype(np.int64) + 4096) << 40) + ((a[:, 2].astype(np.int64) + 4096) << 20) + (a[:, 3].astype(np.int64) + 4096)
    og, oo = np.argsort(key(cg)), np.argsort(key(co))
    m = np.empty(len(cg), dtype=np.int64); m[og] = oo          # gpu row -> oracle row
    return m
m_in = order(cm.sets[ts_in].coords.cpu().numpy(), co_in)
m_out = order(cm.sets[ts_out].coords.cpu().numpy(), co_out)
x_o = torch.zeros(n_in, cin, dtype=torch.float64); x_o[m_in] = x.double()
if ks == 1:
    ref_o = x_o @ w[0].double()
else:
    maps = om.kernel_map(1, 2, ks) if transposed else om.kernel_map(ts_in, ts_out, ks)
    if transposed: maps = [(oo, ii) for ii, oo in maps]
    ref_o = me_cpu._conv_apply(x_o, maps, w.double(), n_out)
scale = shift = res = None
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
assert torch.equal(tc.from_split(s0, cin0), (xd[:, :cin0].bfloat16().float() + (xd[:, :cin0] - xd[:, :cin0].bfloat16().float()).bfloat16().float()))
wp = tc.pack_weights(w.to(dev))
rs = tc.to_split(res_f.to(dev)) if res_f is not None else None
o_split, o_f32 = tc.conv_tc(s0, cin0, s1, cin1, km_nbr, n_out, K, wp, cout, scale.to(dev) if scale is not None else None,
                            shift.to(dev) if shift is not None else None, rs, 'relu' in epi, True, True, None)
torch.cuda.synchronize()
def err(a):
    a = a.double().cpu()
    return float(((a - ref).norm(dim=1) / (ref.norm(dim=1) + 1e-6)).max())
e1, e2 = err(o_f32), err(tc.from_split(o_split, cout))
print('RESULT', mode, cin0, cin1, cout, ks, stride, epi, 'err_f32=%%.3e err_split=%%.3e' %% (e1, e2))
assert e1 < 1e-4 and e2 < 1e-4, (e1, e2)
# scattered fp32 output
perm = torch.randperm(n_out, generator=g).to(dev).int()
_, o_sc = tc.conv_tc(s0, cin0, s1, cin1, km_nbr, n_out, K, wp, cout, None, None, None, False, False, True, perm)
_, o_pl = tc.conv_tc(s0, cin0, s1, cin1, km_nbr, n_out, K, wp, cout, None, None, None, False, False, True, None)
assert torch.equal(o_sc[perm.long()], o_pl)
print('OK')
'''

CASES = [
    # cin0 cin1 cout ks stride epilogue
    (32, 0, 32, 3, 1, 'none'), (96, 0, 96, 3, 1, 'bn+relu'), (96, 0, 96, 3, 1, 'bn+res+relu'), (128, 64, 128, 3, 1, 'bn+relu'),
    (32, 0, 32, 2, 2, 'bn+relu'), (256, 0, 128, 2, -2, 'bn+relu'), (96, 32, 96, 1, 1, 'bn'), (96, 0, 768, 1, 1, 'none'),
    (256, 128, 256, 3, 1, 'bn+relu'), (64, 0, 64, 3, 1, 'none'),
]


def _run(mode, case):
    src = WORKER % {'root': ROOT}
    r = subprocess.run([sys.executable, '-c', src, mode] + [str(v) for v in case], capture_output=True, text=True, timeout=240)
    print(r.stdout[-2000:], r.stderr[-3000:])
    return r


@pytest.mark.parametrize('case', CASES)
def test_conv_tc_cpasync(case):
    r = _run('cpasync', case)
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-500:] + r.stderr[-1500:]


@pytest.mark.parametrize('case', CASES[:2])
def test_conv_tc_row_loads(case):
    r = _run('rows', case)
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-500:] + r.stderr[-1500:]


def test_stem_fused_matches_oracle():
    src = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import synth, tc
from openscene_b200.coords import CoordinateManager
from oracle import me_cpu
dev = torch.device('cuda:0')
c = synth.scene('tiny')
cm = CoordinateManager(torch.from_numpy(c).to(dev))
g = torch.Generator().manual_seed(0)
x = torch.rand(len(c), 3, generator=g)
w = torch.randn(125, 3, 32, generator=g) * 0.1
scale, shift = 0.5 + torch.rand(32, generator=g), torch.randn(32, generator=g) * 0.1
conv = me_cpu.MinkowskiConvolution(3, 32, kernel_size=5, dimension=3).double()
conv.kernel.data = w.double()
ref = torch.relu(conv(me_cpu.SparseTensor(x.double(), torch.from_numpy(c))).F * scale.double() + shift.double())
cs = cm.sets[1].ensure_hash()
xi = x.to(dev)[cm.perm.long()]
o_split, o_f32 = tc.conv_stem(xi, cs.coords, cs.slots, cs.cap, 5, 1, w.to(dev), scale.to(dev), shift.to(dev), True, True, True)
out = o_f32[cm.inv_perm.long()].double().cpu()
e = float(((out - ref).norm(dim=1) / (ref.norm(dim=1) + 1e-6)).max())
print('stem err', e)
assert e < 1e-5
assert float((tc.from_split(o_split, 32) - o_f32).abs().max()) < 1e-4
print('OK')
''' % {'root': ROOT}
    r = subprocess.run([sys.executable, '-c', src], capture_output=True, text=True, timeout=240)
    print(r.stdout[-2000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout


def test_tc_autograd_forward_and_dgrad_match_oracle():
    """SparseConvFunction on 32-multiple channels: forward and dgrad run on the tensor-core kernel (dgrad = the same
    kernel on the transposed map with W^T packed), wgrad on the fp32 kernel.  Against the fp64 oracle's autograd."""
    src = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import me, synth
from oracle import me_cpu
dev = 'cuda:0'
c = synth.scene('tiny')
torch.manual_seed(3)
f = torch.randn(len(c), 32)
fo = f.clone().double().requires_grad_(True)
fg = f.clone().to(dev).requires_grad_(True)
specs = [('c', 32, 64, 3, 1), ('c', 64, 64, 2, 2), ('c', 64, 96, 1, 1), ('t', 96, 32, 2, 2)]
mk = lambda M: [ (M.MinkowskiConvolution if k == 'c' else M.MinkowskiConvolutionTranspose)(i, o, kernel_size=ks, stride=st, dimension=3) for k, i, o, ks, st in specs]
no, ng = mk(me_cpu), mk(me)
for a, b in zip(no, ng):
    b.load_state_dict(a.state_dict()); a.double(); b.to(dev)
xo = me_cpu.SparseTensor(fo, torch.from_numpy(c)); xg = me.SparseTensor(fg, torch.from_numpy(c).to(dev))
for m in no: xo = m(xo)
for m in ng: xg = m(xg)
w = torch.randn(len(c), 32, generator=torch.Generator().manual_seed(9))
(xo.F * w.double()).sum().backward(); (xg.F * w.to(dev)).sum().backward()
rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
e_out = rel(xg.F.detach().cpu().numpy(), xo.F.detach().numpy())
e_gx = rel(fg.grad.cpu().numpy(), fo.grad.numpy())
e_gw = max(rel(b.kernel.grad.cpu().numpy(), a.kernel.grad.numpy()) for a, b in zip(no, ng))
print('err out %%.2e gx %%.2e gw %%.2e' %% (e_out, e_gx, e_gw))
assert e_out < 1e-4 and e_gx < 1e-4 and e_gw < 1e-4
print('OK')
''' % {'root': ROOT}
    r = subprocess.run([sys.executable, '-c', src], capture_output=True, text=True, timeout=240)
    print(r.stdout[-2000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout
