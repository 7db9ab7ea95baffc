"""Forward + backward time of sparse pooling on config2_200k's level-0 coordinate set (2^3 window, stride 2), and one
ResNet18 training step on a batch of two copies of the scene.

Arms, alternated rep by rep:
  identity  the route MinkowskiSumPooling / MinkowskiAvgPooling took before csrc/pool.cu: a sparse convolution with K identity
            kernels (SparseConvFunction; the tensor-core route when C % 32 == 0 and K <= 32), average = sum / count
  pool      the pooling kernels (SparsePoolFunction), average and max
at C = 32, 96 and 256.  Reported per case: median and range in ms, and GB/s against 4 n_in C + 4 n_out C + 4 pairs bytes.
The SM clock is measured on the device between reps (osb_measure_sm_mhz) and the power limit read before the timed region.
Usage: python scripts/bench_pooling.py [--reps 20] [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from openscene_b200 import _cabi as C
    from openscene_b200 import me, resnet, synth
    dev = torch.device('cuda:0')
    pl = power_limit()
    coords = torch.from_numpy(synth.scene('config2_200k')).to(dev)
    x0 = me.SparseTensor(torch.rand(coords.shape[0], 3, device=dev), coords)
    cm = x0.coordinate_manager
    ts = cm.stride(1, 2)
    km = cm.kernel_map(1, ts, 2)
    km.transposed()
    n_in, n_out, pairs = km.n_in, km.n_out, km.num_pairs()
    cnt = (km.nbr >= 0).sum(0).clamp(min=1).float().unsqueeze(1)
    mhz_buf = torch.zeros(1, dtype=torch.float32, device=dev)
    clocks = []

    def identity(x, avg):
        c = x.shape[1]
        eye = torch.eye(c, device=dev).unsqueeze(0).expand(km.K, c, c).contiguous()
        s = me.SparseConvFunction.apply(x, eye, km, n_out)
        return s / cnt if avg else s

    def arm(fn, c):
        x = torch.randn(n_in, c, device=dev, requires_grad=True)
        g = torch.randn(n_out, c, device=dev)

        def run():
            fn(x).backward(g)
            x.grad = None
        return run

    cases = {}
    for c in (32, 96, 256):
        cases[f'avg_c{c}_identity'] = arm(lambda x: identity(x, True), c)
        cases[f'avg_c{c}_pool'] = arm(lambda x: me.SparsePoolFunction.apply(x, km, me.POOL_AVG), c)
        cases[f'max_c{c}_pool'] = arm(lambda x: me.SparsePoolFunction.apply(x, km, me.POOL_MAX), c)
    model = resnet.resnet('ResNet18', 3, 20).to(dev).train()
    opt = torch.optim.SGD(model.parameters(), lr=1e-3)
    two = torch.cat([coords, coords + torch.tensor([1, 0, 0, 0], dtype=coords.dtype, device=dev)])   # a batch of two scenes
    feats = torch.rand(two.shape[0], 3, device=dev)
    labels = torch.tensor([3, 7], device=dev)

    def resnet_step():
        opt.zero_grad(set_to_none=True)
        y = model(me.SparseTensor(feats, two))
        torch.nn.functional.cross_entropy(y, labels).backward()
        opt.step()
    cases['resnet18_train_step'] = resnet_step
    for fn in cases.values():                      # warm-up: kernel maps, weight packs, allocator
        fn(), fn()
    times = {k: [] for k in cases}
    for r in range(args.reps):
        for k, fn in cases.items():                # every arm once per rep, in turn
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
        C.call('osb_measure_sm_mhz', C.ptr(mhz_buf), C.stream_ptr())
        clocks.append(float(mhz_buf.item()))
    res = {'device': torch.cuda.get_device_name(0), 'power_limit_w': pl, 'sm_mhz_median': statistics.median(clocks),
           'sm_mhz_range': [min(clocks), max(clocks)], 'n_in': n_in, 'n_out': n_out, 'pairs': pairs, 'reps': args.reps,
           'cases': {}}
    for k, v in times.items():
        e = {'median_ms': round(statistics.median(v), 4), 'range_ms': [round(min(v), 4), round(max(v), 4)]}
        if k.startswith(('avg', 'max')):
            c = int(k.split('_')[1][1:])
            nbytes = 4 * n_in * c + 4 * n_out * c + 4 * pairs
            e['gb_per_s'] = round(nbytes / (statistics.median(v) * 1e-3) / 1e9, 1)
        res['cases'][k] = e
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_pooling.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
