#!/usr/bin/env python
"""One supervised training step of the 3D baseline (run/train_mink.py: translate, forward, cross-entropy with ignore label 255,
backward, SGD) on a batch of scenes: ``train_mink.train_step`` on the module path against ``train_mink.fused_train_step`` on
``FusedMinkUNet(model, batch_stats=True)``.

    python scripts/bench_train_mink_step.py [--steps K] [--warmup W] [--scenes S] [--kernels] [--out DIR]

Setup: MinkUNet18A with 20 classes, SGD(lr 0.01, momentum 0.9, weight decay 1e-4) as config/scannet/mink.yaml, a batch of
S scenes (synth.scene('config1_50k', seed=i, batch_index=i), i < S, default 8), feats uniform in [0, 1), labels height bands x
x-slabs mod 20 with 10 % set to 255 (as tests/test_gpu_engine_train_ce.py).  Each arm owns a copy of the model and of its
optimiser state; before every step both are restored from the same snapshot and the L2 is flushed (256 MiB memset), outside
the step's CUDA-event pair, and the arms alternate.

Reported: ms per step (min / median / max) of each arm, peak memory per step, the loss difference, the pred agreement and the
largest per-parameter gradient difference (relative to that parameter's largest gradient) after one step from the same state;
the device name, power limit and SM clock.  --kernels also times osb_ce_head_fwd / osb_ce_head_bwd alone (CUDA events over
many launches) at the batch's level-0 size against the bytes a row must move at least, and the torch sequence they replace on
the same rows (split -> fp32, @ w, F.cross_entropy, backward, max(1)).  The JSON line is printed and, with --out, written to
DIR/bench_train_mink_step.json."""
import argparse
import copy
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

CLASSES = 20


def labels_for(coords, c):
    c64 = coords.long()
    lab = ((c64[:, 3] // 8) * 5 + c64[:, 1] // 16) % c
    lab[(c64[:, 1] * 7 + c64[:, 2] * 13 + c64[:, 3] * 3) % 10 == 0] = 255
    return lab


def _time(fn, reps, flush):
    evs = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in evs)
    return {'ms_min': ts[0], 'ms_median': ts[len(ts) // 2], 'ms_max': ts[-1]}


def kernels(n, cin, c, dev, flush, reps=50):
    """osb_ce_head_fwd / _bwd alone on n random rows, and the torch sequence they replace"""
    from openscene_b200 import _cabi as C
    g = torch.Generator().manual_seed(0)
    xf = torch.randn(n, cin, generator=g).to(dev)
    w = (torch.randn(cin, c, generator=g) / cin ** 0.5).to(dev)
    perm = torch.randperm(n, generator=g).to(torch.int32).to(dev)
    lab = torch.randint(0, c, (n,), generator=g)
    lab[torch.rand(n, generator=g) < 0.1] = 255
    lab = lab.to(dev)
    xs = torch.empty((n, 4 * cin), dtype=torch.uint8, device=dev)
    C.call('osb_f32_to_split', C.ptr(xf), n, cin, C.ptr(xs), C.stream_ptr())
    ws_b = C.lib().osb_ce_head_workspace_bytes(n, cin, c)
    ws = torch.empty(ws_b, dtype=torch.uint8, device=dev)
    lse, pred = torch.empty(n, device=dev), torch.empty(n, dtype=torch.int64, device=dev)
    loss, nv, one = torch.empty(1, device=dev), torch.empty(1, dtype=torch.int64, device=dev), torch.ones(1, device=dev)
    dx, dw = torch.empty_like(xs), torch.empty(cin, c, device=dev)
    lib, st = C.lib(), torch.cuda.current_stream().cuda_stream

    def fwd():
        lib.osb_ce_head_fwd(xs.data_ptr(), n, cin, w.data_ptr(), c, perm.data_ptr(), lab.data_ptr(), 1, 255, lse.data_ptr(),
                            pred.data_ptr(), loss.data_ptr(), nv.data_ptr(), ws.data_ptr(), ws_b, st)

    def bwd():
        lib.osb_ce_head_bwd(xs.data_ptr(), n, cin, w.data_ptr(), c, perm.data_ptr(), lab.data_ptr(), 1, 255, lse.data_ptr(),
                            one.data_ptr(), nv.data_ptr(), dx.data_ptr(), dw.data_ptr(), ws.data_ptr(), ws_b, st)
    perm_l = perm.long()
    wt = w.clone().requires_grad_()
    x32 = torch.empty(n, cin, device=dev)

    def torch_seq():
        C.call('osb_split_to_f32', C.ptr(xs), n, cin, C.ptr(x32), C.stream_ptr())
        x = x32.requires_grad_()
        z = x @ wt
        ls = F.cross_entropy(z, lab[perm_l], ignore_index=255)
        ls.backward()
        p = torch.empty(n, dtype=torch.int64, device=dev)
        p[perm_l] = z.detach().max(1)[1]
        x.grad = None
        wt.grad = None
        x32.requires_grad_(False)
    for f_ in (fwd, bwd, torch_seq):
        f_()
    torch.cuda.synchronize()
    t_f, t_b, t_t = _time(fwd, reps, flush), _time(bwd, reps, flush), _time(torch_seq, reps, flush)
    # bytes a row must move: fwd x + row map + label (int64) + lse + pred (int64); bwd x + row map + label + lse + dx
    min_f, min_b = 4 * cin + 4 + 8 + 4 + 8, 4 * cin + 4 + 8 + 4 + 4 * cin
    return {'rows': n, 'cin': cin, 'classes': c, 'fwd': t_f, 'bwd': t_b, 'torch_sequence_fwd_bwd_argmax': t_t,
            'min_bytes_per_row_fwd': min_f, 'min_bytes_per_row_bwd': min_b,
            'fwd_gbps_at_min_traffic': n * min_f / (t_f['ms_median'] * 1e6),
            'bwd_gbps_at_min_traffic': n * min_b / (t_b['ms_median'] * 1e6),
            'kernels_vs_torch_median': t_t['ms_median'] / (t_f['ms_median'] + t_b['ms_median'])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--scenes', type=int, default=8)
    ap.add_argument('--arch', default='MinkUNet18A')
    ap.add_argument('--kernels', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from bench_batch_stats import power_limit_w
    from openscene_b200 import engine, synth, train_mink
    assert torch.cuda.is_available(), "bench_train_mink_step.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    coords = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=i, batch_index=i)) for i in range(args.scenes)])
    labels = labels_for(coords, CLASSES).to(dev)
    coords = coords.to(dev)
    feats = torch.rand(coords.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)
    result = {'metric': 'ms per supervised training step (translate, forward, cross-entropy, backward, SGD)',
              'scene': f'{args.scenes} x config1_50k, {coords.shape[0]} voxels, {CLASSES} classes, '
                       f'{float((labels == 255).float().mean()):.3f} unlabelled',
              'arch': args.arch, 'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w,
              'power_limit_source': power_how, 'steps': args.steps, 'warmup': args.warmup,
              'method': 'weights, buffers and SGD state restored and L2 flushed before every step, outside the CUDA-event pair; '
                        'arms alternate'}

    base = synth.build_model(args.arch, CLASSES, seed=0).train().to(dev)
    m_mod, m_eng = copy.deepcopy(base), copy.deepcopy(base)

    def sgd(m):
        return torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    o_mod, o_eng = sgd(m_mod), sgd(m_eng)
    eng = engine.FusedMinkUNet(m_eng, batch_stats=True)
    train_mink.train_step(m_mod, o_mod, coords, feats, labels)                 # momentum buffers exist in both arms
    train_mink.fused_train_step(eng, o_eng, coords, feats, labels)
    snap_m = copy.deepcopy(base.state_dict())
    snap_o = copy.deepcopy(o_mod.state_dict())

    def restore(m, o):
        with torch.no_grad():
            for k, v in m.state_dict().items():
                v.copy_(snap_m[k])
        o.load_state_dict(snap_o)

    arms = {'module_path': (m_mod, o_mod, lambda: train_mink.train_step(m_mod, o_mod, coords, feats, labels)),
            'engine': (m_eng, o_eng, lambda: train_mink.fused_train_step(eng, o_eng, coords, feats, labels))}
    for _ in range(args.warmup):
        for m, o, fn in arms.values():
            restore(m, o)
            fn()
    # one step from the same state without the update: loss, pred and gradient differences
    losses, preds, grads = {}, {}, {}
    for name, (m, o, _) in arms.items():
        restore(m, o)
        keep = torch.optim.SGD(m.parameters(), lr=0.0)
        keep.step = lambda closure=None: None
        torch.manual_seed(1)
        l, p = (train_mink.train_step(m, keep, coords, feats, labels) if name == 'module_path'
                else train_mink.fused_train_step(eng, keep, coords, feats, labels))
        losses[name], preds[name] = float(l), p
        grads[name] = [q.grad.clone() for q in m.parameters()]
    gdiff = max(float((a - b).abs().max() / (b.abs().max() + 1e-30)) for a, b in zip(grads['engine'], grads['module_path']))
    agree = float((preds['engine'] == preds['module_path']).float().mean())
    del grads, preds
    evs, peak = {n: [] for n in arms}, {}
    gc.collect()
    gc.disable()
    try:
        for i in range(args.steps):
            for name, (m, o, fn) in arms.items():
                restore(m, o)
                flush.zero_()
                torch.cuda.reset_peak_memory_stats(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); fn(); b.record()
                evs[name].append((a, b))
                if i == 0:
                    torch.cuda.synchronize()
                    peak[name] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
            if i in (args.steps // 4, args.steps // 2, (3 * args.steps) // 4):
                sampler.sample()
        torch.cuda.synchronize()
    finally:
        gc.enable()
    result.update({'loss_module': losses['module_path'], 'loss_engine': losses['engine'],
                   'loss_rel_diff': abs(losses['engine'] - losses['module_path']) / abs(losses['module_path']),
                   'pred_agreement': agree, 'max_param_grad_diff_rel_to_max': gdiff, 'peak_mem_gib': peak})
    for name, pairs in evs.items():
        ts = sorted(a.elapsed_time(b) for a, b in pairs)
        result[name] = {'ms_min': ts[0], 'ms_median': ts[len(ts) // 2], 'ms_max': ts[-1]}
    result['speedup_median'] = result['module_path']['ms_median'] / result['engine']['ms_median']
    if args.kernels:
        n0 = eng.last_cm.sets[1].n
        result['kernels'] = kernels(n0, eng.final.cin, CLASSES, dev, flush)
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_train_mink_step.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
