"""Bisect the fixed per-CTA cost of k_conv_tc (tuning aid)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openscene_b200 import synth, tc  # noqa: E402
from openscene_b200.coords import CoordinateManager  # noqa: E402

dev = torch.device('cuda:0')
coords = torch.from_numpy(synth.scene('config2_200k')).to(dev)
cm = CoordinateManager(coords)
n = cm.sets[1].n
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def run(cin, cout, ks, label, clock=False, **dbg):
    nbr, K = (cm.kernel_map(1, 1, ks).nbr, ks ** 3) if ks > 1 else (None, 1)
    x = tc.to_split(torch.randn(n, cin, device=dev))
    w = tc.pack_weights(torch.randn(K, cin, cout, device=dev) * 0.05)
    tc.debug_set_tc(**dbg)
    f32 = cout > 256
    fn = lambda: tc.conv_tc(x, cin, None, 0, nbr, n, K, w, cout, None, None, None, True, not f32, f32, None)
    fn(); torch.cuda.synchronize()
    tot = 0.0
    for _ in range(5):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    msg = f'{label:44s} {cin:3d}->{cout:3d} k{ks}  {1e3 * tot / 5:8.1f} us'
    if clock:
        nt = (n + 127) // 128
        buf = torch.zeros((nt, 8), dtype=torch.int64, device=dev)
        tc.debug_set_clock(buf)
        fn(); torch.cuda.synchronize()
        tc.debug_set_clock(None)
        c = buf.cpu().numpy().astype(np.float64)
        d = np.diff(c[:, :6], axis=1)          # start->setup, ->producers done, ->accum ready, ->stores issued, ->sync
        msg += '  cycles(median): setup %.0f  mainloop-issue %.0f  wait-accum %.0f  epilogue %.0f  final-sync %.0f  total %.0f' % (
            *np.median(d, axis=0), np.median(c[:, 5] - c[:, 0]))
        # concurrency: CTAs alive per SM over time is not observable here; report span of the whole grid instead
        msg += '  grid-span %.0f cycles' % (c[:, 5].max() - c[:, 0].min())
    tc.debug_set_tc(use_gather4=2, smem_budget=227 * 1024, dbg_skip=0, force_split=0, target_ctas=264, pf_dist=0)
    print(msg, flush=True)


run(96, 96, 1, '1x1 full', clock=True)
run(96, 96, 1, '1x1 no main loop', clock=True, dbg_skip=4)
run(96, 96, 1, '1x1 no main loop, no stores', clock=True, dbg_skip=12)
run(96, 96, 1, '1x1 no stores', clock=True, dbg_skip=8)
run(32, 32, 1, '1x1 32->32 (1 stage)', clock=True)
run(96, 96, 3, '3x3x3 full', clock=True)
run(96, 96, 3, '3x3x3 no stores', dbg_skip=8)
run(96, 96, 3, '3x3x3 no main loop (prologue+epilogue)', clock=True, dbg_skip=4)
run(96, 768, 1, 'final full', clock=True)
run(96, 768, 1, 'final no stores', clock=True, dbg_skip=8)
run(96, 768, 1, 'final no main loop', dbg_skip=4)
