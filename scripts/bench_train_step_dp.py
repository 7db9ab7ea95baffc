#!/usr/bin/env python
"""Data-parallel training step on N GPUs: the DistributedDataParallel module path against the fused engine built with
``process_group=dist.group.WORLD``, each with and without its gradient reduction.

    python -m torch.distributed.run --nproc-per-node N scripts/bench_train_step_dp.py [--steps K] [--warmup W] [--out DIR]

Arms, alternated on the same state (weights, buffers and optimiser state restored, L2 flushed with a 256 MiB memset and the
ranks aligned by a barrier before every step, outside the step's CUDA-event pair):
  * ddp:          ``distill.wrap_ddp`` + ``distill.distill_step`` (train_mink: ``train_mink.train_step``);
  * ddp_no_sync:  the same under ``DistributedDataParallel.no_sync()`` (no gradient all-reduce);
  * fused_dp:     ``distill.fused_distill_step`` (``train_mink.fused_train_step``) on the data-parallel engine;
  * fused_local:  the same step on an engine without a process group (no gradient all-reduce).
The difference between an arm and its no-reduction twin is the communication the step exposes.  With N = 1 there is no
DistributedDataParallel wrapper and no reduction: the four arms give the same-build single-GPU baseline.

Workloads: distillation (one synth.scene('config2_200k', seed=rank) per rank, feats = 1, 20,000 supervised rows, 768-d
targets, Adam) on MinkUNet18A and MinkUNet34C; the supervised baseline (MinkUNet18A, 20 classes, a batch of --scenes
config1_50k scenes per rank, labels as tests/test_gpu_engine_train_ce.py, SGD momentum 0.9, weight decay 1e-4).  No random
translation, so every arm sees the same voxels.

Reported per workload and arm: ms per step (min / median / max over ranks and steps), the exposed communication (median of
an arm minus the median of its twin), peak memory (largest over ranks); the device name, power limit, SM clock and N.  Rank 0
prints the JSON line and, with --out, writes it to DIR/bench_train_step_dp_n{N}.json."""
import argparse
import contextlib
import copy
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def _workloads(args, rank, dev):
    from bench_train_mink_step import CLASSES, labels_for
    from openscene_b200 import distill, synth, train_mink
    out = []
    coords = torch.from_numpy(synth.scene('config2_200k', seed=rank)).to(dev)
    feats = torch.ones(coords.shape[0], 3, device=dev)
    g = torch.Generator().manual_seed(rank)
    mask = torch.zeros(coords.shape[0], dtype=torch.bool)
    mask[torch.randperm(coords.shape[0], generator=g)[:args.rows]] = True
    mask = mask.to(dev)
    tgt = torch.randn(args.rows, 768, generator=g).half().to(dev)
    for arch in args.archs.split(','):
        def module_step(m, o):
            return distill.distill_step(m, o, coords, feats, tgt, mask, translate=False)

        def fused_step(e, o):
            return distill.fused_distill_step(e, o, coords, feats, tgt, mask, translate=False)

        def local_step(e, o):                      # fused_distill_step's body: the helper refuses a local engine for N > 1
            loss = distill.distill_loss(e.forward_train(coords, feats, rows=mask), tgt)
            o.zero_grad()
            loss.backward()
            o.step()
        out.append((f'distill {arch}', f'config2_200k seed=rank, {coords.shape[0]} voxels on rank {rank}, {args.rows} rows',
                    lambda a=arch: synth.build_model(a, 768, seed=0),
                    lambda ps: torch.optim.Adam(ps, lr=1e-3), module_step, fused_step, local_step))
    cs = [torch.from_numpy(synth.scene('config1_50k', seed=rank * args.scenes + i, batch_index=i)) for i in range(args.scenes)]
    c2 = torch.cat(cs)
    lab = labels_for(c2, CLASSES).to(dev)
    c2 = c2.to(dev)
    f2 = torch.rand(len(c2), 3, generator=torch.Generator().manual_seed(2)).to(dev)

    def module_step2(m, o):
        return train_mink.train_step(m, o, c2, f2, lab, translate=False)

    def fused_step2(e, o):
        return train_mink.fused_train_step(e, o, c2, f2, lab, translate=False)

    def local_step2(e, o):
        loss, _ = e.forward_train_ce(c2, f2, lab, ignore_index=255)
        o.zero_grad()
        loss.backward()
        o.step()
    out.append(('train_mink MinkUNet18A', f'{args.scenes} config1_50k scenes per rank, {len(c2)} voxels on rank {rank}, '
                f'{CLASSES} classes', lambda: synth.build_model('MinkUNet18A', CLASSES, seed=0),
                lambda ps: torch.optim.SGD(ps, lr=0.01, momentum=0.9, weight_decay=1e-4), module_step2, fused_step2, local_step2))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--archs', default='MinkUNet18A,MinkUNet34C')
    ap.add_argument('--rows', type=int, default=20000)
    ap.add_argument('--scenes', type=int, default=8)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    assert torch.cuda.is_available(), "bench_train_step_dp.py needs CUDA devices (no CPU fallback)"
    from openscene_b200 import distill, engine
    local = int(os.environ.get('LOCAL_RANK', 0))
    if local >= torch.cuda.device_count():
        raise SystemExit(f"bench_train_step_dp.py: one device per process: local rank {local} with "
                         f"{torch.cuda.device_count()} visible")
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    if 'RANK' not in os.environ:
        os.environ.update(RANK='0', WORLD_SIZE='1', MASTER_ADDR='127.0.0.1', MASTER_PORT='29531')
    dist.init_process_group('nccl', device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    sampler = None
    if rank == 0:
        from bench import ClockSampler
        from bench_batch_stats import power_limit_w
        power_w, power_how = power_limit_w(local)
        sampler = ClockSampler(local, dev)
        result = {'metric': 'ms per data-parallel training step (forward, loss, backward with gradient all-reduce, optimiser)',
                  'gpus': world, 'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w,
                  'power_limit_source': power_how, 'steps': args.steps, 'warmup': args.warmup,
                  'method': 'weights, buffers and optimiser state restored, L2 flushed and ranks aligned by a barrier before '
                            'every step, outside the CUDA-event pair; arms alternate; ms over all ranks and steps',
                  'workloads': {}}

    for name, scene, build, make_opt, module_step, fused_step, local_step in _workloads(args, rank, dev):
        base = build().train().to(dev)
        m_ddp, m_eng = copy.deepcopy(base), copy.deepcopy(base)
        m_ddp = distill.wrap_ddp(m_ddp, device=dev)
        o_ddp, o_eng = make_opt(m_ddp.parameters()), make_opt(m_eng.parameters())
        e_dp = engine.FusedMinkUNet(m_eng, batch_stats=True, process_group=dist.group.WORLD)
        e_local = engine.FusedMinkUNet(m_eng, batch_stats=True)
        no_sync = m_ddp.no_sync if hasattr(m_ddp, 'no_sync') else contextlib.nullcontext
        module_step(m_ddp, o_ddp)                                   # optimiser state exists in every arm
        fused_step(e_dp, o_eng)
        snap_m = copy.deepcopy(base.state_dict())
        snap_o = copy.deepcopy(o_ddp.state_dict())

        def restore(m, o):
            with torch.no_grad():
                for v, s in zip(m.state_dict().values(), snap_m.values()):
                    v.copy_(s)
            o.load_state_dict(snap_o)

        def ddp_no_sync():
            with no_sync():
                module_step(m_ddp, o_ddp)
        arms = {'ddp': (m_ddp, o_ddp, lambda: module_step(m_ddp, o_ddp)),
                'ddp_no_sync': (m_ddp, o_ddp, ddp_no_sync),
                'fused_dp': (m_eng, o_eng, lambda: fused_step(e_dp, o_eng)),
                'fused_local': (m_eng, o_eng, lambda: local_step(e_local, o_eng))}
        for _ in range(args.warmup):
            for m, o, fn in arms.values():
                restore(m, o)
                fn()
        evs, peak = {n: [] for n in arms}, {}
        gc.collect()
        gc.disable()
        try:
            for i in range(args.steps):
                for arm, (m, o, fn) in arms.items():
                    restore(m, o)
                    flush.zero_()
                    torch.cuda.reset_peak_memory_stats(dev)
                    torch.cuda.synchronize(dev)
                    dist.barrier()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); fn(); b.record()
                    evs[arm].append((a, b))
                    if i == 0:
                        torch.cuda.synchronize(dev)
                        peak[arm] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
                if sampler is not None and i in (args.steps // 4, args.steps // 2, (3 * args.steps) // 4):
                    sampler.sample()
            torch.cuda.synchronize(dev)
        finally:
            gc.enable()
        ms = torch.tensor([[a.elapsed_time(b) for a, b in evs[arm]] for arm in arms], device=dev)
        mem = torch.tensor([peak[arm] for arm in arms], device=dev)
        all_ms = [torch.empty_like(ms) for _ in range(world)]
        all_mem = [torch.empty_like(mem) for _ in range(world)]
        dist.all_gather(all_ms, ms)
        dist.all_gather(all_mem, mem)
        if rank == 0:
            ms, mem = torch.stack(all_ms).cpu(), torch.stack(all_mem).amax(0).cpu()
            rec = {'scene': scene}
            for j, arm in enumerate(arms):
                t = ms[:, j].flatten().sort().values
                rec[arm] = {'ms_min': float(t[0]), 'ms_median': float(t[len(t) // 2]), 'ms_max': float(t[-1]),
                            'peak_mem_gib': float(mem[j])}
            rec['exposed_comm_ms_ddp'] = rec['ddp']['ms_median'] - rec['ddp_no_sync']['ms_median']
            rec['exposed_comm_ms_fused'] = rec['fused_dp']['ms_median'] - rec['fused_local']['ms_median']
            rec['speedup_fused_dp_over_ddp'] = rec['ddp']['ms_median'] / rec['fused_dp']['ms_median']
            result['workloads'][name] = rec
        del e_dp, e_local, m_ddp, m_eng, o_ddp, o_eng, base
        torch.cuda.empty_cache()
    if rank == 0:
        result['clocks'] = sampler.stop()
        line = json.dumps(result)
        print(line)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, f'bench_train_step_dp_n{world}.json'), 'w') as f:
                f.write(line + '\n')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
