"""Bit-exact probes of the documented tensor-core arithmetic.

Operands lie on a dyadic grid small enough that every partial sum an fp32 accumulator can form is an exact multiple of the
grid below 2^24 grid units, so the result cannot depend on summation order, split-K, or the rounding of the accumulator: it
must be BIT-IDENTICAL to an exact fp64 evaluation of the documented arithmetic (include/osb200.h, DESIGN.md section 3):
  * forward (osb_conv_fwd_tc, the persistent chain, osb_convtr_fwd_tc): hi*Whi + hi*Wlo + lo*Whi -- no lo*Wlo;
  * weight gradient (osb_conv_wgrad_tc): all four quadrants (hi + lo)(hi + lo).
Split rows are written directly as bf16 halves, so lo-only rows (hi = 0) occur; weights go through the library's own
packing, so each is chosen with Whi = bf16_rn(w) and Wlo = w - Whi.  The epilogue uses power-of-two scales and on-grid shifts
and residuals, so it is exact too, and the split output must equal split(fp32 output).  Each probe computes its own budget
(log2 of the largest sum of |terms| over the grid) and asserts it, so an inexact case is never compared.

Shapes: the distinct (cin0, cin1, cout, K, map kind) the fused engine launches for all ten architectures (harvested with the
CPU launch recorder of tests/test_engine_train_plan_cpu.py), output row tails 1 / 127 / 128 / 129, a weight gradient whose
row ranges end in a partial range, the padded 5^3 stem gradient, a 1x1x1 gradient over a row selection, and single layers
of the persistent kernel on 148 and 3 CTAs and with forced split-K."""
import os
import subprocess
import sys

import pytest
import torch

from tests.test_engine_plan_cpu import SCENES
from tests.test_engine_train_plan_cpu import _i, _run as _train_run, recorded  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import math, sys, torch
sys.path.insert(0, %(root)r)
from openscene_b200 import synth, tc, _cabi as C
from openscene_b200.coords import CoordinateManager
from tests import replay_ref as R
grid_, fsplit = int(sys.argv[1]), int(sys.argv[2])
cases = eval(sys.argv[3])
if grid_:
    tc.tuning_set('chain_grid', grid_); tc.tuning_set('chain_force_split', fsplit)
dev = torch.device('cuda:0')
g = torch.Generator(device=dev).manual_seed(0)
cm = CoordinateManager(torch.from_numpy(synth.scene('tiny')).to(dev))
cm.stride(1, 2)
n0, n1 = cm.sets[1].n, cm.sets[2].n
down = cm.kernel_map(1, 2, 2)
sel = (torch.arange(n0, device=dev) * 7 %% n0)[: n0 // 3].sort().values.int().view(1, -1).contiguous()
MAPS = {'3': (cm.kernel_map(1, 1, 3).nbr, n0), '5': (cm.kernel_map(1, 1, 5).nbr, n0), 'down': (down.nbr, n0),
        'up': (down.transposed().nbr, n1), 'id': (None, n0), 'sel': (sel, n0),
        'selT': (R.transpose_map(sel, n0).int().contiguous(), sel.shape[1])}

def pick(shape, vals, p):
    v = torch.tensor(vals, dtype=torch.float32, device=dev)
    x = v[torch.randint(len(vals), shape, device=dev, generator=g)]
    return x * (torch.rand(shape, device=dev, generator=g) < p)

def rows(n, c, p, sh=-2, hi_on=True):
    """split rows: hi in {-1,0,1}, lo in {-1,0,1} 2^sh, independent (lo-only entries occur)"""
    hi = pick((n, c), [-1., 1.], p if hi_on else 0.)
    lo = pick((n, c), [-1., 1.], p) * 2.0 ** sh
    return R.split_encode(hi.bfloat16(), lo.bfloat16()), hi.double(), lo.double()

def weights(K, ci, co):
    """w = Whi + Wlo with Whi in {0, +-1, +-2, +-3} = bf16_rn(w), Wlo in {-1, 0, 1} 2^-10"""
    whi = pick((K, ci, co), [-3., -2., -1., 1., 2., 3.], 0.8)
    wlo = pick((K, ci, co), [-1., 1.], 0.7) * 2.0 ** -10 * (whi != 0)
    w = whi + wlo
    assert torch.equal(w.bfloat16().float(), whi) and torch.equal((w - w.bfloat16().float()).bfloat16().float(), wlo)
    return w, whi.double(), wlo.double()

def check_out(tag, o_split, o_f32, ref, cout):
    ok32 = torch.equal(o_f32.double(), ref)
    oks = o_split is None or torch.equal(o_split, R.split_of(o_f32))
    if not (ok32 and oks):
        d = (o_f32.double() - ref).abs()
        i = int(d.argmax())
        print('MISMATCH', tag, 'max |diff| %%.6g at row %%d col %%d (got %%.9g, exact %%.9g), split_ok %%s'
              %% (float(d.max()), i // cout, i %% cout, float(o_f32.view(-1)[i]), float(ref.view(-1)[i]), oks), flush=True)
        raise SystemExit(1)

def fwd(c0, c1, cout, K, kind, transposed, path, epi, n_tail=None, lo_only=False):
    nbr, n_in = MAPS[kind]
    n_out = nbr.shape[1] if nbr is not None else n_in
    if n_tail is not None:
        nbr, n_out = nbr[:, :n_tail].contiguous(), n_tail
    cin = c0 + c1
    p = min(0.5, 2.0 ** 8 / (K * cin))
    s0, h0, l0 = rows(n_in, c0, p, hi_on=not lo_only)
    s1, h1, l1 = rows(n_in, c1, p) if c1 else (None, None, None)
    hi, lo = (torch.cat([h0, h1], 1), torch.cat([l0, l1], 1)) if c1 else (h0, l0)
    w, whi, wlo = weights(K, cin, cout)
    ref = sum(R.conv(a, nbr, n_out, b, want_abs=False)[0] for a, b in ((hi, whi), (hi, wlo), (lo, whi)))
    terms = R.conv(hi.abs() + lo.abs(), nbr, n_out, whi.abs() + wlo.abs(), want_abs=False)[0]
    scale = shift = res = None
    if epi:
        scale = 2.0 ** torch.randint(-1, 2, (cout,), device=dev, generator=g).float()
        shift = torch.randint(-16, 17, (cout,), device=dev, generator=g).float() / 16
        res, rh, rl = rows(n_out, cout, 0.5, sh=-12)
        ref, _ = R.epilogue(ref, terms, scale, shift, rh + rl, relu=True)
    bits = R.exact_budget_bits(terms * 2 + 2, 2.0 ** -13)
    assert bits < 24, ('budget', bits)
    wk = w.transpose(1, 2).contiguous() if transposed else w
    if path == 'tc':
        wp = tc.pack_weights(wk, transpose_w=transposed)
        o_split, o_f32 = tc.conv_tc(s0, c0, s1, c1, nbr, n_out, K, wp, cout, scale, shift, res, bool(epi), True, True, None)
    else:
        wt = tc.pack_weight_tiles(wk, transpose_w=transposed)
        o_split, o_f32 = tc.conv_chain_single(s0, c0, s1, c1, nbr, n_out, K, wt, cout, scale, shift, res, bool(epi), True, True, None)
    torch.cuda.synchronize()
    check_out(('fwd', path, c0, c1, cout, K, kind, transposed, epi, n_tail, lo_only), o_split, o_f32, ref, cout)
    return bits

def convtr(cin, cout, path):
    d = down.nbr
    p = min(0.5, 2.0 ** 8 / cin)
    s, hi, lo = rows(n1, cin, p)
    w, whi, wlo = weights(8, cin, cout)
    ref = sum(R.convtr(a, d, b, n0)[0] for a, b in ((hi, whi), (hi, wlo), (lo, whi)))
    terms = R.convtr(hi.abs() + lo.abs(), d, whi.abs() + wlo.abs(), n0)[0]
    scale = 2.0 ** torch.randint(-1, 2, (cout,), device=dev, generator=g).float()
    shift = torch.randint(-16, 17, (cout,), device=dev, generator=g).float() / 16
    ref, _ = R.epilogue(ref, terms, scale, shift, relu=True)
    bits = R.exact_budget_bits(terms * 2 + 1, 2.0 ** -13)
    assert bits < 24, ('budget', bits)
    wide = w.permute(1, 0, 2).reshape(1, cin, 8 * cout).contiguous()
    if path == 'tc':
        o_split = torch.empty((n0, 4 * cout), dtype=torch.uint8, device=dev)
        o_f32 = torch.empty((n0, cout), dtype=torch.float32, device=dev)
        C.call('osb_convtr_fwd_tc', C.ptr(s), cin, n1, C.ptr(d), 8, C.ptr(tc.pack_weights(wide)), cout, C.ptr(scale), C.ptr(shift),
               1, C.ptr(o_split), C.ptr(o_f32), 0, C.stream_ptr())
    else:
        o_split, o_f32 = tc.conv_chain_single(s, cin, None, 0, None, n1, 1, tc.pack_weight_tiles(wide), 8 * cout, scale, shift, None,
                                              True, True, True, None, cmap=d, cmap_cout=cout, n_rows_out=n0)
    torch.cuda.synchronize()
    check_out(('convtr', path, cin, cout), o_split, o_f32, ref, cout)
    return bits

def wgrad(cin, cout, K, kind, n_rows=None, lo_only=False):
    if n_rows is not None:                     # identity map over n_rows rows (row-range plans)
        nbr, n_in, n_out = None, n_rows, n_rows
    else:
        nbr, n_in = MAPS[kind]
        n_out = nbr.shape[1] if nbr is not None else n_in
    xs, xh, xl = rows(n_in, cin, 0.5, sh=-3)
    gs, gh, gl = rows(n_out, cout, 0.5, sh=-3, hi_on=not lo_only)
    ref = R.wgrad(xh + xl, nbr, gh + gl, K)[0]
    terms = R.wgrad(xh.abs() + xl.abs(), nbr, gh.abs() + gl.abs(), K)[0]
    bits = R.exact_budget_bits(terms, 2.0 ** -6)
    assert bits < 24, ('budget', bits)
    gw = tc.conv_wgrad_tc(xs, cin, n_in, nbr, n_out, K, gs, cout)
    torch.cuda.synchronize()
    check_out(('wgrad', cin, cout, K, kind, n_rows, lo_only, 'n_rs', R.wgrad_plan(n_out, K, cin, cout)), None, gw.view(-1, cout),
              ref.view(-1, cout), cout)
    return bits

worst_bits = 0.0
for case in cases:
    op, args = case[0], case[1:]
    b = {'fwd': fwd, 'convtr': convtr, 'wgrad': wgrad}[op](*args)
    worst_bits = max(worst_bits, b)
print('EXACT %%d probes bit-identical, largest budget 2^%%.2f of 2^24' %% (len(cases), worst_bits), flush=True)
print('OK')
'''


def _run(cases, grid=0, fsplit=0, timeout=900):
    r = subprocess.run([sys.executable, '-c', WORKER % {'root': ROOT}, str(grid), str(fsplit), repr(cases)],
                       capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def _kind(K, nbr, n_in, n_out):
    if K == 1:
        return 'id' if not nbr else ('sel' if n_out < n_in else 'selT')
    if K == 8:
        return 'down' if n_out < n_in else 'up'
    return {27: '3', 125: '5'}[K]


def harvest(rec):
    """distinct launch shapes of forward_train + backward over the ten architectures (CPU recorder, no device work)"""
    from openscene_b200 import engine, minkunet, synth
    fwd, wg, ctr = set(), set(), set()
    n = rec.n = SCENES['tiny']
    for arch in sorted(minkunet.ARCHS):
        model = synth.build_model(arch, 768, seed=0).train()
        eng = engine.FusedMinkUNet(model, batch_stats=True)
        rec.calls.clear()
        out = _train_run(eng, n, torch.arange(n[0]) % 7 == 0)
        nf = len(rec.calls)
        out.sum().backward()
        for j, (name, a) in enumerate(rec.calls):
            a = [_i(x) for x in a]
            if name == 'osb_conv_fwd_tc':
                fwd.add((a[1], a[4], a[10], a[8], _kind(a[8], a[6], a[2], a[7]), j >= nf))
            elif name == 'osb_conv_wgrad_tc':
                wg.add((a[1], a[7], a[5], _kind(a[5], a[3], a[2], a[4])))
            elif name == 'osb_convtr_fwd_tc':
                ctr.add((a[1], a[6]))
    return sorted(fwd), sorted(wg), sorted(ctr)


def test_exact_engine_shapes(recorded):
    fwd, wg, ctr = harvest(recorded)
    assert len(fwd) > 20 and len(wg) > 20 and ctr
    wkinds, fkinds = {w[3] for w in wg}, {f[4] for f in fwd}
    assert {'5', 'up', 'down', 'sel', '3', 'id'} <= wkinds                 # the padded stem gradient, the head over a selection
    assert {'selT', 'sel', 'up', 'down', '3', 'id'} <= fkinds and any(f[1] for f in fwd)
    cases = [('fwd', c0, c1, co, K, kd, T, 'tc', not T) for (c0, c1, co, K, kd, T) in fwd]
    cases += [('wgrad', ci, co, K, kd) for (ci, co, K, kd) in wg]
    cases += [('convtr', ci, co, 'tc') for (ci, co) in ctr]
    print('harvested', len(fwd), 'forward / dgrad,', len(wg), 'wgrad,', len(ctr), 'transposed shapes')
    _run(cases)


def test_exact_tails_and_row_plans():
    cases = []
    for n in (1, 127, 128, 129):
        cases += [('fwd', 96, 0, 96, 27, '3', False, 'tc', True, n), ('fwd', 32, 32, 64, 27, '3', True, 'tc', False, n),
                  ('wgrad', 96, 96, 1, 'id', n)]
    cases += [('wgrad', 32, 32, 1, 'id', 10000), ('wgrad', 64, 160, 1, 'id', 77777),        # n_rs > 1, partial last range
              ('wgrad', 32, 32, 125, '5'),                                                   # the stem's padded gradient
              ('wgrad', 96, 768, 1, 'sel'), ('wgrad', 96, 96, 1, 'sel', None, True),         # head over a row selection
              ('fwd', 96, 0, 96, 27, '3', False, 'tc', True, None, True),                    # lo-only activations
              ('fwd', 768, 0, 96, 1, 'selT', True, 'tc', False)]
    _run(cases)


def test_row_range_cases_are_partial():
    """the identity wgrad probes above really exercise several row ranges with a partial last one"""
    from tests import replay_ref as R
    for (n, ci, co) in ((10000, 32, 32), (77777, 64, 160)):
        n_rs, rpr = R.wgrad_plan(n, 1, ci, co)
        assert n_rs > 1 and n % rpr != 0


CHAIN = [('fwd', 32, 0, 32, 27, '3', False, 'chain', True), ('fwd', 96, 0, 96, 27, '3', False, 'chain', True),
         ('fwd', 128, 64, 128, 27, '3', False, 'chain', True), ('fwd', 256, 128, 256, 27, '3', False, 'chain', False),
         ('fwd', 32, 0, 64, 8, 'down', False, 'chain', True), ('fwd', 96, 0, 96, 8, 'up', True, 'chain', False),
         ('fwd', 96, 32, 96, 1, 'id', False, 'chain', True), ('fwd', 96, 0, 768, 1, 'id', False, 'chain', False),
         ('fwd', 384, 0, 384, 27, '3', False, 'chain', True), ('fwd', 96, 0, 96, 27, '3', False, 'chain', True, 129),
         ('convtr', 256, 128, 'chain'), ('convtr', 96, 96, 'chain')]


@pytest.mark.parametrize('grid,fsplit', [(148, 0), (3, 0), (148, 4), (5, 3)])
def test_exact_chain_single_layers(grid, fsplit):
    _run(CHAIN if fsplit == 0 else [c for c in CHAIN if c[0] == 'fwd'], grid, fsplit)
