"""Per-item time of the training loaders' aug=True chain: the device path (openscene_b200.augmentation.DeviceItemAugmenter,
host draws and syncs included) against the NumPy / SciPy host chain (tests/augment_ref.py, the reference's calls), for
the config1_50k and config2_200k point clouds; plus one fused_train_step fed by eight device items.

Usage: python scripts/bench_augment.py --out DIR [--reps 5]
Prints one JSON line and writes it to DIR/bench_augment.json."""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np
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


def timed(fn, reps, sync):
    ts = []
    for r in range(reps):
        random.seed(r)
        np.random.seed(r)
        sync()
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_augment.py needs a CUDA device"
    from openscene_b200 import augmentation, engine, synth, train_mink
    from tests import augment_ref as A
    sync = torch.cuda.synchronize
    res = {'metric': 'ms per training item (aug=True), median', 'device': torch.cuda.get_device_name(0),
           'power_limit_w': power_limit(), 'reps': args.reps, 'scenes': {}}
    it = augmentation.DeviceItemAugmenter(voxel_size=0.05, input_color=True)
    for name in ('config1_50k', 'config2_200k'):
        pts, _ = synth.scene_points(name, seed=0)
        pts = pts.astype(np.float32)
        n = len(pts)
        rng = np.random.RandomState(0)
        feats = ((rng.rand(n, 3).astype(np.float32) * 2 - 1) + 1.) * 127.5
        labels = rng.randint(0, 20, n).astype(np.uint8)
        mask_full = rng.rand(n) < 0.6
        blob = {'feat': torch.from_numpy(rng.randn(int(mask_full.sum()), 768).astype(np.float16)),
                'mask_full': torch.from_numpy(mask_full)}
        row = {'points': n}
        for kind in ('point', 'fused'):
            if kind == 'point':
                dev = lambda: it.point(pts, feats, labels)                           # noqa: E731
                host = lambda: A.point_item(pts, feats, labels, input_color=True)    # noqa: E731
            else:
                dev = lambda: it.fused(pts, feats, labels, blob)                     # noqa: E731
                host = lambda: A.fused_item(pts, feats, labels, blob, input_color=True)  # noqa: E731
            dev()                                                                     # warm-up
            with np.errstate(invalid='ignore', divide='ignore'):
                row[kind] = {'device_ms': round(timed(dev, args.reps, sync), 2),
                             'host_chain_ms': round(timed(host, max(2, args.reps // 2), lambda: None), 2)}
        res['scenes'][name] = row
    # one training step on eight device-built items
    random.seed(0)
    np.random.seed(0)
    parts = []
    for b in range(8):
        pts, _ = synth.scene_points('config1_50k', seed=b)
        n = len(pts)
        rng = np.random.RandomState(b)
        parts.append(it.point(pts, rng.rand(n, 3) * 255, rng.randint(0, 20, n).astype(np.uint8), batch_index=b))
    coords, feats_b, labels_b = (torch.cat([p[i] for p in parts]) for i in range(3))
    model = synth.build_model('MinkUNet18A', 20, seed=0).train().cuda()
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    train_mink.fused_train_step(eng, opt, coords, feats_b, labels_b)
    step = timed(lambda: train_mink.fused_train_step(eng, opt, coords, feats_b, labels_b), args.reps, sync)
    res['fused_train_step'] = {'voxels': int(coords.shape[0]), 'ms': round(step, 2)}
    os.makedirs(args.out, exist_ok=True)
    line = json.dumps(res)
    with open(os.path.join(args.out, 'bench_augment.json'), 'w') as f:
        f.write(line + '\n')
    print(line)


if __name__ == '__main__':
    main()
