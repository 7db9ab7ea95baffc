"""Weight gradient on tensor cores (csrc/conv_wgrad_tc.cu: MN-major UMMA operands, four-quadrant split product,
deterministic two-kernel reduction) against the fp64 oracle's autograd.  Tolerance 1e-4 relative to the largest entry of
each offset's gradient (observed ~1e-6).  The CUDA-core osb_conv_wgrad_f32 runs alongside and must stay within its
per-element bound (tests/replay_ref.py, DESIGN.md section 2)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import synth, tc, _cabi as C
from openscene_b200.coords import CoordinateManager
from tests import replay_ref as R
dev = torch.device('cuda:0')
cases = eval(sys.argv[1])
for (scene, cin, cout, ks, stride) in cases:
    c = synth.scene(scene) if scene != 'cloud' else synth.random_cloud(700, 16, seed=1)
    cm = CoordinateManager(torch.from_numpy(c).to(dev))
    ts_out = 1
    if stride == 2:
        cm.stride(1, 2); ts_out = 2
    n_in, n_out = cm.sets[1].n, cm.sets[ts_out].n
    K = ks ** 3
    nbr = cm.kernel_map(1, ts_out, ks).nbr if ks > 1 else None
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(n_in, cin, device=dev, generator=g)
    go = torch.randn(n_out, cout, device=dev, generator=g)
    # reference: fp64 gather + matmul per offset
    ref = torch.zeros(K, cin, cout, dtype=torch.float64, device=dev)
    for k in range(K):
        if nbr is None:
            ref[k] = x.double().t() @ go.double()
        else:
            o = (nbr[k] >= 0).nonzero()[:, 0]
            ref[k] = x.double()[nbr[k][o].long()].t() @ go.double()[o]
    gw = tc.conv_wgrad_tc(tc.to_split(x), cin, n_in, nbr, n_out, K, tc.to_split(go), cout)
    torch.cuda.synchronize()
    err = float(((gw.double() - ref).abs().amax(dim=(1, 2)) / (ref.abs().amax(dim=(1, 2)) + 1e-30)).max())
    gw32 = torch.empty_like(gw)
    C.call('osb_conv_wgrad_f32', C.ptr(x), C.ptr(nbr), n_out, K, C.ptr(go), cin, cout, C.ptr(gw32), C.stream_ptr())
    torch.cuda.synchronize()
    err32 = float(((gw32.double() - ref).abs().amax(dim=(1, 2)) / (ref.abs().amax(dim=(1, 2)) + 1e-30)).max())
    # the CUDA-core kernel within its per-element bound (tests/replay_ref.py): (depth + 3) 2^-24 sum |x||g|
    _, A = R.wgrad(x.double(), nbr, go.double(), K)
    c32 = R.c_fma(R.f32_wgrad_depth(R.f32_dispatch('wgrad', cin, cout, K, nbr is not None), n_out))
    frac32 = R.worst(gw32, ref, A, c32) / c32
    assert frac32 <= 1.0, frac32
    gw2 = tc.conv_wgrad_tc(tc.to_split(x), cin, n_in, nbr, n_out, K, tc.to_split(go), cout)
    print('RESULT', scene, cin, cout, ks, stride, 'n_out', n_out, 'err_tc=%%.3e err_f32_kernel=%%.3e (%%.3f of its bound)' %% (err, err32, frac32), flush=True)
    assert err < 1e-4, err
    assert torch.equal(gw, gw2)                       # fixed-order reduction: bit-reproducible
print('OK')
'''

CASES = [('tiny', 32, 32, 3, 1), ('tiny', 96, 96, 3, 1), ('tiny', 64, 128, 3, 1), ('tiny', 256, 256, 3, 1), ('tiny', 192, 96, 3, 1),
         ('tiny', 32, 64, 2, 2), ('cloud', 96, 768, 1, 1), ('cloud', 128, 96, 1, 1), ('config1_50k', 96, 96, 3, 1)]


def test_wgrad_tc_matches_fp64_reference():
    src = WORKER % {'root': ROOT}
    r = subprocess.run([sys.executable, '-c', src, repr(CASES)], capture_output=True, text=True, timeout=600)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]
