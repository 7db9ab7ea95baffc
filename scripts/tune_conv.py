"""GPU micro-benchmark of the tensor-core sparse-conv kernel on the config-2 scene (tuning aid, not a bench line).
Prints microseconds per launch for a few shapes under different pipeline settings."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openscene_b200 import synth, tc  # noqa: E402
from openscene_b200.coords import CoordinateManager  # noqa: E402

dev = torch.device('cuda:0')
coords = torch.from_numpy(synth.scene(sys.argv[1] if len(sys.argv) > 1 else 'config2_200k')).to(dev)
cm = CoordinateManager(coords)
ts = [1]
for _ in range(4):
    ts.append(cm.stride(ts[-1], 2))
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


HOT = False


def timeit(fn, reps=5):
    fn(); torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        if not HOT:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    return 1e3 * tot / reps


def case(level, cin, cout, ks, label, **dbg):
    t = ts[level]
    n = cm.sets[t].n
    if ks == 1:
        nbr, K = None, 1
    else:
        km = cm.kernel_map(t, t, ks)
        nbr, K = km.nbr, km.K
    x = tc.to_split(torch.randn(n, cin, device=dev))
    w = tc.pack_weights(torch.randn(K, cin, cout, device=dev) * 0.05)
    tc.debug_set_tc(**dbg)
    f32 = cout > 256
    us = timeit(lambda: tc.conv_tc(x, cin, None, 0, nbr, n, K, w, cout, None, None, None, True, not f32, f32, None))
    tc.debug_set_tc(use_gather4=2, smem_budget=227 * 1024, dbg_skip=0, force_split=0, target_ctas=132, pf_dist=0, small_nt=0, min_stages=3, lazy=1)
    print(f'{label:46s} L{level} n={n:7d} {cin:3d}->{cout:3d} k{ks}  {us:9.1f} us', flush=True)


B2, B1 = 112 * 1024, 226 * 1024
if len(sys.argv) > 2 and sys.argv[2] == 'lazy':
    for (lvl, cin, cout, ks) in ((0, 96, 96, 3), (0, 128, 96, 3), (0, 96, 96, 1), (0, 96, 768, 1), (1, 64, 64, 3), (1, 192, 96, 3), (2, 128, 128, 3), (3, 256, 256, 3), (4, 256, 256, 3)):
        case(lvl, cin, cout, ks, 'smem index prologue', lazy=0)
        case(lvl, cin, cout, ks, 'lazy per-offset index fetch', lazy=2)
    sys.exit(0)
if len(sys.argv) > 2 and sys.argv[2] == 'occ':
    B3, B4 = 75 * 1024, 56 * 1024
    for (lvl, cin, cout, ks) in ((1, 64, 64, 3), (1, 192, 96, 3), (1, 96, 96, 3), (0, 96, 96, 3), (0, 128, 96, 3), (0, 96, 96, 1), (2, 128, 128, 3), (0, 32, 32, 2)):
        case(lvl, cin, cout, ks, 'default smem budget')
        case(lvl, cin, cout, ks, '75 KB smem budget, 2 stages', smem_budget=B3, min_stages=2)
        case(lvl, cin, cout, ks, '56 KB smem budget, 2 stages', smem_budget=B4, min_stages=2)
    sys.exit(0)
if len(sys.argv) > 2 and sys.argv[2] == 'small':
    for lvl in (2, 3, 4):
        c = {2: 128, 3: 256, 4: 256}[lvl]
        for snt in (0, 128, 64):
            for tgt in (132, 264):
                case(lvl, c, c, 3, f'L{lvl} small_nt={snt} target={tgt}', small_nt=snt, target_ctas=tgt)
        case(lvl, c, c, 1, f'L{lvl} 1x1 small_nt=0', small_nt=0)
        case(lvl, c, c, 1, f'L{lvl} 1x1 small_nt=64', small_nt=64)
    sys.exit(0)
if len(sys.argv) > 2 and sys.argv[2] == 'pf':
    for hot in (False, True):
        HOT = hot
        for pf in (0, 132, 264, 396, 528):
            case(0, 96, 96, 3, f'hot={hot} pf_dist={pf}', pf_dist=pf)
        case(0, 96, 96, 3, f'hot={hot} pf 132, budget B1', pf_dist=132, smem_budget=B1)
        case(0, 128, 96, 3, f'hot={hot} 128->96 pf 296', pf_dist=296)
        case(0, 96, 96, 1, f'hot={hot} 1x1 pf 0', pf_dist=0)
        case(0, 96, 96, 1, f'hot={hot} 1x1 pf 296', pf_dist=296)
        case(0, 96, 768, 1, f'hot={hot} final pf 0', pf_dist=0)
        case(0, 96, 768, 1, f'hot={hot} final pf 296', pf_dist=296)
    sys.exit(0)
case(0, 96, 96, 3, 'base (default smem budget, cp.async)')
case(0, 96, 96, 3, '1 CTA/SM deep pipeline', smem_budget=B1)
case(0, 96, 96, 3, 'no A gathers (timing only)', dbg_skip=1)
case(0, 96, 96, 3, 'no B loads (timing only)', dbg_skip=2)
case(0, 96, 96, 3, 'no A, no B (MMA + epilogue only)', dbg_skip=3)
case(0, 96, 96, 3, 'no A, 1 CTA/SM', dbg_skip=1, smem_budget=B1)
case(0, 96, 96, 3, 'no B, 1 CTA/SM', dbg_skip=2, smem_budget=B1)
case(0, 128, 96, 3, 'base 128->96')
case(0, 96, 768, 1, 'final 96->768 fp32 out')
case(0, 96, 96, 1, '1x1x1 96->96')
for lvl, tag in ((1, 'L1 64->64'), (2, 'L2'), (3, 'L3'), (4, 'L4')):
    c = {1: 64, 2: 128, 3: 256, 4: 256}[lvl]
    case(lvl, c, c, 3, f'{tag} heuristic split')
    case(lvl, c, c, 3, f'{tag} no split', force_split=1)
    case(lvl, c, c, 3, f'{tag} target 592 CTAs', target_ctas=592)
    case(lvl, c, c, 3, f'{tag} target 132 CTAs', target_ctas=132)
