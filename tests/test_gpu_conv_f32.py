"""The fp32 CUDA-core convolutions of csrc/conv_f32.cu, called through their C entry points, against fp64.

Every shape is run twice (tests/replay_ref.py holds the reference, the bound and the dispatch restatement):
  * bound: random operands whose rows span 17 binades; every output element must satisfy
    |y - y^| <= (depth + 3) 2^-24 A with A = sum |x||W| (wgrad: sum |x||g|) and the depth of the kernel's launch plan
    (``R.f32_depth``: K cin FMAs for the forwards, a row chunk plus its atomic adds for the weight gradients);
  * exact probe: dyadic operands (features {0, +-1, +-2} 2^-3, weights and gradients {0, +-1, +-2, +-3} 2^-4) whose sums
    stay below 2^24 units of 2^-7, asserted before comparing, so every fp32 partial and every atomic add is exact in any order
    and the result must equal fp64 bit for bit.  A dropped row, chunk or offset that hides below a depth-linear bound at
    200k rows shows here; the atomic weight gradients must also be bit-reproducible on these operands.
Outputs are views into NaN-filled buffers: every element of the result must be written and nothing around it touched.
Inputs come plain, offset by one float (the scalar A-load branch) and with a row stride of cin + 3 whose unused columns hold
NaN, so any read of them poisons the result.  Maps: the library's own cubic maps on the 197k-voxel config2_200k scene (the
7^3 one from the independent ``R.neighbour_map``), truncated to the first n_out output rows, and synthetic maps for K that is
not a cube (random input rows, 30 % absent, a 64-row tile absent for every third offset, one offset with no pairs).
The workers run in child processes, as in test_gpu_conv_exact.py."""
import itertools
import os
import subprocess
import sys

import pytest

from tests import replay_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import math, sys, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import synth, _cabi as C
from openscene_b200.coords import CoordinateManager
from tests import replay_ref as R
cases = eval(sys.argv[1])
dev = torch.device('cuda:0')
g = torch.Generator(device=dev).manual_seed(0)
NAN, PRE, POST = float('nan'), 32, 45
cm = CoordinateManager(torch.from_numpy(synth.scene('config2_200k')).to(dev))
cm.stride(1, 2)
N0 = cm.sets[1].n
CUBES = {'c3': (27, lambda: cm.kernel_map(1, 1, 3).nbr), 'c5': (125, lambda: cm.kernel_map(1, 1, 5).nbr),
         'c7': (343, lambda: R.neighbour_map(cm.sets[1].coords, 7, 1).int().contiguous()),
         'down': (8, lambda: cm.kernel_map(1, 2, 2).nbr)}
_maps = {}

def holes(nbr):
    """a 64-row tile with no neighbour for every third offset, and one offset without any pair"""
    nbr = nbr.clone()
    K, n = nbr.shape
    if K > 1 and n > 128:
        nbr[::3, 64:128] = -1
        nbr[K // 2] = -1
    return nbr

def get_map(kind, K, n_out):
    """(nbr or None, n_in, n_out); n_out 'scene': every row of the 197k-voxel scene"""
    if n_out == 'scene' and kind not in CUBES and kind != 'h3':
        n_out = N0
    if kind == 'id':
        assert K == 1
        return None, n_out, n_out
    if kind in ('c3', 'c5', 'c7', 'down', 'h3'):
        base = 'c3' if kind == 'h3' else kind
        assert CUBES[base][0] == K, (kind, K)
        if base not in _maps:
            _maps[base] = CUBES[base][1]()
        nbr = _maps[base]
        n_out = nbr.shape[1] if n_out == 'scene' else n_out
        assert n_out <= nbr.shape[1], (kind, n_out)
        nbr = nbr[:, :n_out].contiguous()
        return (holes(nbr) if kind == 'h3' else nbr), N0, n_out
    if kind == 'sel':                          # K = 1 over a sparse selection of rows
        assert K == 1
        n_in = 3 * n_out + 7
        return torch.randperm(n_in, device=dev, generator=g)[:n_out].sort().values.int().view(1, -1).contiguous(), n_in, n_out
    assert kind == 'syn'
    n_in = n_out + 100
    nbr = torch.randint(n_in, (K, n_out), device=dev, generator=g, dtype=torch.int32)
    nbr[torch.rand((K, n_out), device=dev, generator=g) < 0.3] = -1
    return holes(nbr).contiguous(), n_in, n_out

def guarded(n):
    buf = torch.full((PRE + n + POST,), NAN, device=dev)
    return buf, buf[PRE:PRE + n]

def guard_ok(buf, n):
    return bool(torch.isnan(buf[:PRE]).all()) and bool(torch.isnan(buf[PRE + n:]).all())

def operands(shape, mode, kind):
    """'x': features, 'w': weights / output gradients"""
    if mode == 'exact':
        return R.probe_x(shape, g, dev) if kind == 'x' else R.probe_w(shape, g, dev)
    if kind == 'x':
        return R.binade_rows(shape[0], shape[1], 8, g, dev)
    return R.binade_rows(shape[0] * shape[1], shape[2], 2, g, dev).view(shape) if len(shape) == 3 else R.binade_rows(*shape, 2, g, dev)

worst, budget, seen = {}, 0.0, set()

def judge(tag, kernel, mode, y, ref, A, depth, buf, n):
    global budget
    if not guard_ok(buf, n):
        print('GUARD', tag, 'wrote outside its output', flush=True); raise SystemExit(1)
    if bool(torch.isnan(y).any()):
        print('UNWRITTEN', tag, int(torch.isnan(y).sum()), 'elements left NaN (or NaN read)', flush=True); raise SystemExit(1)
    if mode == 'exact':
        bits = R.exact_budget_bits(A, R.PROBE_GRID)
        assert bits < 24, ('budget', tag, bits)
        budget = max(budget, bits)
        if not torch.equal(y.double(), ref):
            d = (y.double() - ref).abs()
            i = int(d.argmax())
            print('MISMATCH', tag, 'max |diff| %%.6g at flat %%d (got %%.9g, exact %%.9g)'
                  %% (float(d.max()), i, float(y.reshape(-1)[i]), float(ref.reshape(-1)[i])), flush=True)
            raise SystemExit(1)
    else:
        c = R.c_fma(depth)
        fr = R.worst(y, ref, A, c) / c
        worst[kernel] = max(worst.get(kernel, 0.0), fr)
        if not fr <= 1.0:
            print('BOUND', tag, 'uses %%.3f of (depth %%d + 3) 2^-24 A' %% (fr, depth), flush=True); raise SystemExit(1)
    seen.add(kernel)

def fwd(n_out, cin, cout, K, kind, T, layout, mode):
    nbr, n_in, n_out = get_map(kind, K, n_out)
    vals = operands((n_in, cin), mode, 'x')
    ld = cin
    if layout == 'ld':                        # row stride cin + 3, the unused columns NaN
        ld = cin + 3
        xb = torch.full((n_in, ld), NAN, device=dev); xb[:, :cin] = vals; xp = xb
    elif layout == 'unaligned':               # offset by one float: the scalar A-load branch
        xb = torch.full((n_in * cin + 1,), NAN, device=dev); xp = xb[1:]; xp.copy_(vals.view(-1))
    else:
        xp = vals.contiguous()
    w = operands((K, cin, cout), mode, 'w')
    wk = w.transpose(1, 2).contiguous() if T else w
    kernel = R.f32_dispatch('fwd', cin, cout, K, nbr is not None, ld, T)
    buf, out = guarded(n_out * cout)
    C.call('osb_conv_fwd_f32', C.ptr(xp), ld, C.ptr(nbr), n_out, K, C.ptr(wk), cin, cout, int(T), C.ptr(out), C.stream_ptr())
    torch.cuda.synchronize()
    ref, A = R.conv(vals.double(), nbr, n_out, w.double())
    judge(('fwd', n_out, cin, cout, K, kind, T, layout, mode, kernel), kernel, mode, out.view(n_out, cout), ref, A,
          R.f32_depth(kernel, K, cin, n_out), buf, n_out * cout)

def wgrad(n_out, cin, cout, K, kind, mode):
    nbr, n_in, n_out = get_map(kind, K, n_out)
    x = operands((n_in, cin), mode, 'x').contiguous()
    go = operands((n_out, cout), mode, 'w').contiguous()
    kernel = R.f32_dispatch('wgrad', cin, cout, K, nbr is not None)
    n = K * cin * cout
    runs = []
    for _ in range(2 if mode == 'exact' else 1):
        buf, gw = guarded(n)
        C.call('osb_conv_wgrad_f32', C.ptr(x), C.ptr(nbr), n_out, K, C.ptr(go), cin, cout, C.ptr(gw), C.stream_ptr())
        torch.cuda.synchronize()
        runs.append((buf, gw))
    ref, A = R.wgrad(x.double(), nbr, go.double(), K)
    tag = ('wgrad', n_out, cin, cout, K, kind, mode, kernel)
    for buf, gw in runs:
        judge(tag, kernel, mode, gw.view(K, cin, cout), ref, A, R.f32_depth(kernel, K, cin, n_out), buf, n)
    if len(runs) == 2 and not torch.equal(runs[0][1].view(torch.int32), runs[1][1].view(torch.int32)):
        print('NONDETERMINISTIC', tag, flush=True); raise SystemExit(1)

def gather(n_out, c, kind):
    n_in = {'perm': n_out, 'repeat': 7, 'empty': 5}[kind]
    x = torch.randn((n_in, c), device=dev, generator=g)
    idx = (torch.randperm(n_in, device=dev, generator=g) if kind == 'perm'
           else torch.randint(n_in, (n_out,), device=dev, generator=g)).int()
    buf, out = guarded(n_out * c)
    C.call('osb_gather_rows_f32', C.ptr(x), C.ptr(idx), n_out, c, C.ptr(out), C.stream_ptr())
    torch.cuda.synchronize()
    ref = x[idx.long()].reshape(-1)
    if not guard_ok(buf, n_out * c) or not torch.equal(out.view(torch.int32), ref.view(torch.int32)):
        print('MISMATCH gather', n_out, c, kind, flush=True); raise SystemExit(1)
    seen.add('gather')

NAMES = {'fwd_thin': 'k_conv_fwd_thin', 'fwd_generic': 'k_conv_fwd_f32', 'wgrad_thin': 'k_conv_wgrad_thin',
         'wgrad_generic': 'k_conv_wgrad_f32'}

def dispatch(entry, cin, cout, K, has_nbr, ld_extra, T):
    """the kernel the library really launches (torch.profiler) is the one the restatement names"""
    n_out = 9
    nbr = get_map('syn', K, n_out)[0] if has_nbr else None
    n_in = n_out + 100 if has_nbr else n_out
    x = torch.zeros((n_in, cin + ld_extra), device=dev)
    want = R.f32_dispatch(entry, cin, cout, K, has_nbr, cin + ld_extra, T)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        if entry == 'fwd':
            w, out = torch.zeros((K, cin, cout), device=dev), torch.empty((n_out, cout), device=dev)
            C.call('osb_conv_fwd_f32', C.ptr(x), cin + ld_extra, C.ptr(nbr), n_out, K, C.ptr(w), cin, cout, int(T), C.ptr(out),
                   C.stream_ptr())
        else:
            go, gw = torch.zeros((n_out, cout), device=dev), torch.empty((K, cin, cout), device=dev)
            C.call('osb_conv_wgrad_f32', C.ptr(x), C.ptr(nbr), n_out, K, C.ptr(go), cin, cout, C.ptr(gw), C.stream_ptr())
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()} | {e.key for e in prof.key_averages()}
    names = {nm for nm in names if 'k_conv_' in nm}
    got = {k for k, v in NAMES.items() if any(v + '<' in nm or v + '(' in nm for nm in names)}
    if got != {want}:
        print('DISPATCH', (entry, cin, cout, K, has_nbr, ld_extra, T), 'restated', want, 'launched', sorted(names), flush=True)
        raise SystemExit(1)
    seen.add(want)

for case in cases:
    op, args = case[0], case[1:]
    if op in ('fwd', 'wgrad'):
        for mode in ('bound', 'exact'):
            (fwd if op == 'fwd' else wgrad)(*args, mode)
    else:
        {'gather': gather, 'dispatch': dispatch}[op](*args)
print('KERNELS', ','.join(sorted(seen)))
print('WORST', ' '.join('%%s=%%.4f' %% kv for kv in sorted(worst.items())), 'of the bound; largest exact budget 2^%%.2f of 2^24'
      %% budget, flush=True)
print('OK')
'''


def _run(cases, timeout=1200):
    r = subprocess.run([sys.executable, '-c', WORKER % {'root': ROOT}, repr(cases)], capture_output=True, text=True,
                       timeout=timeout)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    return [l for l in r.stdout.splitlines() if l.startswith('KERNELS ')][-1].split()[1].split(',')


def _kernels(cases):
    """what the restated dispatch says the cases reach"""
    out = set()
    for c in cases:
        if c[0] == 'fwd':
            _, n, cin, cout, K, kind, T, layout = c
            out.add(R.f32_dispatch('fwd', cin, cout, K, kind != 'id', cin + 3 if layout == 'ld' else cin, T))
        elif c[0] == 'wgrad':
            _, n, cin, cout, K, kind = c
            out.add(R.f32_dispatch('wgrad', cin, cout, K, kind != 'id'))
    return out


_FWD_KINDS = [(1, 'id'), (1, 'sel'), (8, 'down'), (27, 'c3'), (125, 'c5'), (343, 'c7'), (27, 'h3'), (33, 'syn')]


def fwd_generic_cases():
    cases = []
    for i, (cin, cout) in enumerate(itertools.product((1, 3, 5, 15, 16, 17, 33, 96, 255), (1, 3, 20, 63, 64, 65, 129, 768))):
        K, kind = _FWD_KINDS[i % 8]
        n = (1, 63, 64, 65, 4097)[i % 5]
        cases.append(('fwd', n, cin, cout, K, kind, (i // 8) % 2, ('plain', 'unaligned', 'ld')[i % 3]))
    cases += [('fwd', 'scene', 96, 96, 27, 'c3', 0, 'plain'),          # the fp32 yardstick of test_gpu_fullsize.py
              ('fwd', 'scene', 17, 45, 27, 'h3', 1, 'ld'), ('fwd', 'scene', 96, 20, 1, 'sel', 0, 'unaligned')]
    return cases


def fwd_thin_cases():
    cases, ns = [], (1, 8, 9, 8448, 8449)
    kinds = [(1, 'sel'), (8, 'down'), (27, 'c3'), (31, 'syn'), (32, 'syn'), (33, 'syn'), (125, 'c5')]
    for i, (cin, (K, kind)) in enumerate(itertools.product((1, 2, 3, 4), kinds)):
        cases.append(('fwd', ns[i % 5], cin, 32, K, kind, 0, 'plain' if i % 3 else 'unaligned'))
    cases += [('fwd', 8449, 1, 32, 343, 'c7', 0, 'plain'), ('fwd', 9, 2, 32, 343, 'c7', 0, 'unaligned'),
              ('fwd', 8448, 3, 32, 256, 'syn', 0, 'plain'),          # exactly 96 KiB of weights in shared memory
              ('fwd', 8449, 3, 32, 257, 'syn', 0, 'plain'),          # one offset more: the generic kernel
              ('fwd', 8449, 3, 32, 125, 'c5', 0, 'ld'),              # a row stride > cin: the generic kernel
              ('fwd', 'scene', 3, 32, 125, 'c5', 0, 'plain')]        # the stem of distill_step on the 197k scene
    return cases


def wgrad_generic_cases():
    cases, ns = [], (1, 15, 16, 17, 4095, 4096, 4097, 3 * 4096 + 1)
    for i, (cin, cout) in enumerate(itertools.product((63, 64, 65, 129), repeat=2)):
        K, kind = ((1, 'id'), (27, 'c3'))[i // 8]
        cases.append(('wgrad', ns[i % 8], cin, cout, K, kind))
    cases += [('wgrad', 4097, 3, 32, 129, 'syn'), ('wgrad', 8449, 2, 32, 343, 'c7'),     # beyond the thin kernel's 128 offsets
              ('wgrad', 4096, 5, 32, 27, 'c3'), ('wgrad', 12289, 3, 31, 125, 'c5'),
              ('wgrad', 'scene', 65, 63, 27, 'c3'), ('wgrad', 'scene', 96, 20, 1, 'id')]
    return cases


def wgrad_thin_cases():
    cases, ns = [], (1, 127, 128, 129, 67584, 67585)
    kinds = [(1, 'sel'), (7, 'syn'), (8, 'syn'), (9, 'syn'), (125, 'c5'), (127, 'syn'), (128, 'syn')]
    for i, (cin, (K, kind)) in enumerate(itertools.product((1, 2, 3, 4), kinds)):
        cases.append(('wgrad', ns[i % 6], cin, 32, K, kind))
    cases += [('wgrad', 129, 3, 32, 8, 'down'), ('wgrad', 67585, 3, 32, 125, 'c5'), ('wgrad', 67585, 4, 32, 128, 'syn'),
              ('wgrad', 'scene', 3, 32, 125, 'c5')]                    # the stem gradient of distill_step
    return cases


def test_fwd_generic():
    cases = fwd_generic_cases()
    assert _kernels(cases) == {'fwd_generic'}
    assert set(_run(cases)) == {'fwd_generic'}


def test_fwd_thin():
    cases = fwd_thin_cases()
    assert _kernels(cases) == {'fwd_thin', 'fwd_generic'}
    assert R.f32_dispatch('fwd', 3, 32, 256, True) == 'fwd_thin' and R.f32_dispatch('fwd', 3, 32, 257, True) == 'fwd_generic'
    assert set(_run(cases)) == _kernels(cases)


def test_wgrad_generic():
    cases = wgrad_generic_cases()
    assert _kernels(cases) == {'wgrad_generic'}
    assert set(_run(cases)) == {'wgrad_generic'}


def test_wgrad_thin():
    cases = wgrad_thin_cases()
    assert _kernels(cases) == {'wgrad_thin'}
    assert R.thin_wgrad_grid(67585) == 528 and -(-67585 // R.THIN_WG_ROWS) == 529   # one block walks two chunks
    assert set(_run(cases)) == {'wgrad_thin'}


def test_gather_rows():
    cases = [('gather', n, c, kind) for c in (1, 3, 32, 768) for (n, kind) in ((4099, 'perm'), (1000, 'repeat'), (0, 'empty'))]
    assert _run(cases) == ['gather']


def test_dispatch_restatement_matches_the_library():
    cases = []
    for cin, K in ((1, 768), (2, 384), (3, 256), (4, 192)):                # the 96 KiB shared-memory ceiling of the thin forward
        cases += [('dispatch', 'fwd', cin, 32, K, True, 0, 0), ('dispatch', 'fwd', cin, 32, K + 1, True, 0, 0)]
    cases += [('dispatch', 'fwd', 3, 32, 27, True, 3, 0), ('dispatch', 'fwd', 3, 32, 27, True, 0, 1),
              ('dispatch', 'fwd', 3, 31, 27, True, 0, 0), ('dispatch', 'fwd', 5, 32, 27, True, 0, 0),
              ('dispatch', 'fwd', 3, 32, 1, False, 0, 0)]
    for cin in (1, 4, 5):
        cases += [('dispatch', 'wgrad', cin, 32, 128, True, 0, 0), ('dispatch', 'wgrad', cin, 32, 129, True, 0, 0)]
    cases += [('dispatch', 'wgrad', 3, 33, 27, True, 0, 0), ('dispatch', 'wgrad', 3, 32, 1, False, 0, 0)]
    assert set(_run(cases)) == {'fwd_thin', 'fwd_generic', 'wgrad_thin', 'wgrad_generic'}
