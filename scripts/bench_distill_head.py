#!/usr/bin/env python
"""The distillation step's head on the fused engine: ``distill.fused_distill_step`` (tensor-core head launch, torch's cosine
loss chain on the fp32 [M, 768] rows, the split conversion of their gradient, head wgrad and dgrad) against
``distill.fused_cosine_step`` (osb_cos_head_fwd / osb_cos_head_bwd), both with ``optim.Adam`` bound to the engine; with
--loss l1, ``fused_distill_step(loss_type='l1')`` (torch's L1 chain) against ``distill.fused_l1_step`` (osb_l1_head_fwd /
osb_l1_head_bwd).

    python scripts/bench_distill_head.py [--loss cosine|l1] [--steps K] [--warmup W] [--out DIR]

Workloads: one synth.scene('config2_200k') with 20,000 supervised rows on MinkUNet18A and MinkUNet34C (the config3_distill
shape), and 8 synth.scene('config1_50k') scenes with 20,000 rows each (160,000 rows) on MinkUNet18A (the one-GPU ScanNet /
Matterport batch of 8).  Each arm owns a copy of the model and its Adam state; before every step both are restored in place
from the same snapshot and re-packed, and the L2 is flushed (256 MiB memset), outside the step's CUDA-event pair; the arms
alternate.

Head alone: from the trunk output of one forward, the old head (osb_conv_fwd_tc on the rows, distill_loss forward and backward,
osb_f32_to_split, osb_conv_wgrad_tc, the dgrad osb_conv_fwd_tc) against the two new launches, CUDA events around just that
work, L2 flushed before each, alternating.  Kernel counts per step and per head come from torch.profiler in a separate run.

Reported per workload: ms per step and per head (min / median / max), kernels per step and per head, peak memory per step, the
loss difference and the largest per-parameter gradient difference (relative to that parameter's largest gradient) after one
step from the same state; and the device name, power limit and SM clocks sampled during the run.  The JSON line is printed
and, with --out, written to DIR/bench_distill_head.json (--loss l1: DIR/bench_distill_head_l1.json)."""
import argparse
import copy
import functools
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import torch  # noqa: E402

WORKLOADS = [('config2_200k x1, 18A', 'MinkUNet18A', 'config2_200k', 1),
             ('config2_200k x1, 34C', 'MinkUNet34C', 'config2_200k', 1),
             ('config1_50k x8, 18A', 'MinkUNet18A', 'config1_50k', 8)]


def _data(scene, k, rows, dev):
    from openscene_b200 import synth
    coords = torch.cat([torch.from_numpy(synth.scene(scene, seed=s, batch_index=s)) for s in range(k)])
    g = torch.Generator().manual_seed(0)
    mask = torch.zeros(coords.shape[0], dtype=torch.bool)
    off = 0
    for s in range(k):                                       # `rows` supervised rows per scene
        n_s = int((coords[:, 0] == s).sum())
        mask[off + torch.randperm(n_s, generator=g)[:rows]] = True
        off += n_s
    m = int(mask.sum())
    return (coords.to(dev), torch.ones(coords.shape[0], 3, device=dev), mask.to(dev),
            torch.randn(m, 768, generator=g).half().to(dev))


def _stats(ts):
    ts = sorted(ts)
    return {'ms_min': ts[0], 'ms_median': ts[len(ts) // 2], 'ms_max': ts[-1]}


def _kernels(fn):
    """CUDA kernels one call of fn launches (torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'Memset' not in e.name
               and 'Memcpy' not in e.name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rows', type=int, default=20000)
    ap.add_argument('--workloads', default='0,1,2')
    ap.add_argument('--out', default=None)
    ap.add_argument('--loss', choices=('cosine', 'l1'), default='cosine')
    args = ap.parse_args()

    from bench import ClockSampler
    from bench_batch_stats import power_limit_w
    from openscene_b200 import _cabi as C
    from openscene_b200 import distill, engine, optim, synth, tc
    assert torch.cuda.is_available(), "bench_distill_head.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)
    new = args.loss                                                  # the arm and head names: cosine_step / l1_step, ...
    result = {'metric': f'ms per distillation step (translate, forward, {new} loss, backward, bound Adam) and per head',
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w, 'power_limit_source': power_how,
              'steps': args.steps, 'warmup': args.warmup, 'rows_per_scene': args.rows,
              'method': 'weights, buffers and Adam state restored in place, re-packed, L2 flushed before every step and every '
                        'head call, outside the CUDA-event pair; arms alternate',
              'workloads': {}}

    for wi in [int(x) for x in args.workloads.split(',')]:
        label, arch, scene, k = WORKLOADS[wi]
        coords, feats, mask, tgt = _data(scene, k, args.rows, dev)
        base = synth.build_model(arch, 768, seed=0).train().to(dev)
        arms = {}
        new_step = distill.fused_cosine_step if new == 'cosine' else distill.fused_l1_step
        for name, step in (('distill_step', functools.partial(distill.fused_distill_step, loss_type=new)),
                           (f'{new}_step', new_step)):
            m = copy.deepcopy(base)
            eng = engine.FusedMinkUNet(m, batch_stats=True)
            o = optim.Adam(m.parameters(), lr=1e-3)
            o.bind(eng)
            step(eng, o, coords, feats, tgt, mask)                  # Adam state exists
            arms[name] = (m, eng, o, step)
        snap_m = copy.deepcopy(base.state_dict())
        snap_o = {name: [{kk: (v.clone() if torch.is_tensor(v) else v) for kk, v in o.state[p].items()} for p in m.parameters()]
                  for name, (m, eng, o, _) in arms.items()}

        def restore(name):
            m, eng, o, _ = arms[name]
            with torch.no_grad():
                for kk, v in m.state_dict().items():
                    v.copy_(snap_m[kk])
                for p, st in zip(m.parameters(), snap_o[name]):
                    for kk, v in st.items():
                        if torch.is_tensor(v):
                            o.state[p][kk].copy_(v)
                        else:
                            o.state[p][kk] = v
            o.repack_bound()

        def run(name):
            m, eng, o, step = arms[name]
            return step(eng, o, coords, feats, tgt, mask)

        for _ in range(args.warmup):
            for name in arms:
                restore(name)
                run(name)
        # one step from the same state without the update
        losses, grads = {}, {}
        for name, (m, eng, o, step) in arms.items():
            restore(name)
            keep = torch.optim.SGD(m.parameters(), lr=0.0)
            keep.step = lambda closure=None: None
            torch.manual_seed(1)
            losses[name] = float(step(eng, keep, coords, feats, tgt, mask))
            grads[name] = [p.grad.clone() for p in m.parameters()]
        gdiff = max(float((a - b).abs().max() / (b.abs().max() + 1e-30))
                    for a, b in zip(grads[f'{new}_step'], grads['distill_step']))
        del grads
        evs, peak = {n: [] for n in arms}, {}
        gc.collect()
        gc.disable()
        try:
            for i in range(args.steps):
                for name in arms:
                    restore(name)
                    flush.zero_()
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats(dev)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); run(name); b.record()
                    evs[name].append((a, b))
                    if i == 0:
                        torch.cuda.synchronize()
                        peak[name] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
                if i in (args.steps // 4, args.steps // 2, (3 * args.steps) // 4):
                    sampler.sample()
            torch.cuda.synchronize()
        finally:
            gc.enable()
        rec = {'rows': int(mask.sum()), 'voxels': int(coords.shape[0]), 'arch': arch,
               'loss_distill_step': losses['distill_step'], f'loss_{new}_step': losses[f'{new}_step'],
               'loss_rel_diff': abs(losses[f'{new}_step'] - losses['distill_step']) / abs(losses['distill_step']),
               'max_param_grad_diff_rel_to_max': gdiff, 'peak_mem_gib': peak}
        for name, pairs in evs.items():
            rec[name] = _stats([a.elapsed_time(b) for a, b in pairs])
        rec['step_speedup_median'] = rec['distill_step']['ms_median'] / rec[f'{new}_step']['ms_median']
        rec['kernels_per_step'] = {}
        for name in arms:
            restore(name)
            rec['kernels_per_step'][name] = _kernels(lambda: run(name))

        # ---- the head alone, on the trunk output of one forward
        m, eng, o, _ = arms['distill_step']
        restore('distill_step')
        out = eng.forward_train(coords, feats, rows=mask)
        gr = out.grad_fn.graph
        kind, nd = gr.tape[-1]
        assert kind == 'head'
        (src, cin, n0), = nd.srcs
        sel = gr.keep[1]
        mm, cc = sel.shape[0], nd.cv.cout
        fin = eng.final
        lib = C.lib()
        stream = torch.cuda.current_stream().cuda_stream
        pk = tc.pack_weights(fin.mod.kernel.detach().unsqueeze(0), transpose_w=True)
        dx = torch.empty((n0, 4 * cin), dtype=torch.uint8, device=dev)
        gsplit = torch.empty((mm, 4 * cc), dtype=torch.uint8, device=dev)
        dw = torch.empty((cin, cc), device=dev)
        wg_ws = torch.empty(max(lib.osb_conv_wgrad_tc_workspace_bytes(mm, 1, cin, cc), 256), dtype=torch.uint8, device=dev)
        cos_ws = torch.empty(getattr(lib, f'osb_{"cos" if new == "cosine" else "l1"}_head_workspace_bytes')(mm, cin, cc),
                             dtype=torch.uint8, device=dev)
        state = torch.empty((mm, 3), dtype=torch.float64, device=dev)
        signs = torch.empty((mm, cc // 16), dtype=torch.int32, device=dev)
        loss = torch.empty((), device=dev)
        one = torch.ones((), device=dev)

        def old_head():
            f = torch.empty((mm, cc), dtype=torch.float32, device=dev)
            C.check(eng._fn(src, cin, n0, 0, 0, 0, nd.nbr_f, mm, 1, fin.wpack_a, cc, 0, 0, 0, 0, 0, f.data_ptr(), 0, eng._ws_a,
                            eng._ws_bytes, eng._flags, stream), 'osb_conv_fwd_tc')
            f.requires_grad_()
            distill.distill_loss(f, tgt, new).backward()
            C.call('osb_f32_to_split', C.ptr(f.grad), mm, cc, C.ptr(gsplit), C.stream_ptr())
            C.check(lib.osb_conv_wgrad_tc(src, cin, n0, nd.nbr_f, mm, 1, gsplit.data_ptr(), cc, dw.data_ptr(), wg_ws.data_ptr(),
                                          wg_ws.numel(), stream), 'osb_conv_wgrad_tc')
            C.check(lib.osb_conv_fwd_tc(gsplit.data_ptr(), cc, mm, 0, 0, 0, nd.nbr_b, n0, 1, pk.data_ptr(), cin, 0, 0, 0, 0,
                                        dx.data_ptr(), 0, 0, eng._ws_a, eng._ws_bytes, 0, stream), 'osb_conv_fwd_tc')

        def new_head():
            C.check(lib.osb_cos_head_fwd(src, n0, cin, fin.w3.data_ptr(), cc, sel.data_ptr(), mm, tgt.data_ptr(),
                                         state.data_ptr(), loss.data_ptr(), cos_ws.data_ptr(), cos_ws.numel(), stream),
                    'osb_cos_head_fwd')
            C.check(lib.osb_cos_head_bwd(src, n0, cin, fin.w3.data_ptr(), cc, sel.data_ptr(), mm, tgt.data_ptr(),
                                         state.data_ptr(), one.data_ptr(), dx.data_ptr(), dw.data_ptr(), cos_ws.data_ptr(),
                                         cos_ws.numel(), stream), 'osb_cos_head_bwd')

        def l1_head():
            C.check(lib.osb_l1_head_fwd(src, n0, cin, fin.w3.data_ptr(), cc, sel.data_ptr(), mm, tgt.data_ptr(), signs.data_ptr(),
                                        loss.data_ptr(), cos_ws.data_ptr(), cos_ws.numel(), stream), 'osb_l1_head_fwd')
            C.check(lib.osb_l1_head_bwd(src, n0, cin, fin.w3.data_ptr(), cc, sel.data_ptr(), mm, signs.data_ptr(), one.data_ptr(),
                                        dx.data_ptr(), dw.data_ptr(), cos_ws.data_ptr(), cos_ws.numel(), stream),
                    'osb_l1_head_bwd')

        heads = {'old_head': old_head, f'{new}_head': new_head if new == 'cosine' else l1_head}
        for fn in heads.values():
            for _ in range(3):
                fn()
        hev, hpeak = {n: [] for n in heads}, {}
        for i in range(max(args.steps, 20)):
            for name, fn in heads.items():
                flush.zero_()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                base_mem = torch.cuda.memory_allocated(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); fn(); b.record()
                hev[name].append((a, b))
                if i == 0:
                    torch.cuda.synchronize()
                    hpeak[name] = (torch.cuda.max_memory_allocated(dev) - base_mem) / 2 ** 30
        torch.cuda.synchronize()
        for name, pairs in hev.items():
            rec[name] = _stats([a.elapsed_time(b) for a, b in pairs])
        rec['head_speedup_median'] = rec['old_head']['ms_median'] / rec[f'{new}_head']['ms_median']
        rec['head_extra_mem_gib'] = hpeak
        rec['kernels_per_head'] = {name: _kernels(fn) for name, fn in heads.items()}
        rec[f'{new}_head_share_of_step'] = rec[f'{new}_head']['ms_median'] / rec[f'{new}_step']['ms_median']
        del out, gr, nd
        result['workloads'][label] = rec
        print(label, json.dumps(rec), flush=True)
        del arms, base
        torch.cuda.empty_cache()
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = 'bench_distill_head.json' if new == 'cosine' else 'bench_distill_head_l1.json'
        with open(os.path.join(args.out, name), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
