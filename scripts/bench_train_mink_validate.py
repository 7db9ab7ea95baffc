#!/usr/bin/env python
"""One run/train_mink.py validation (validate(), :349-393) on the eval engine, the reference's torch tail after the forward
against openscene_b200.train_mink.DeviceMinkValidation, and train()'s per-step meters (torch against DeviceTrainMeter).

    python scripts/bench_train_mink_validate.py [--scenes N] [--reps R] [--archs A,B] [--train-steps K] [--out DIR]

Scenes: N (default 16) synthetic rooms, half synth.scene('config1_50k', seed=i) and half 'config2_200k', each with 1.5 points
per voxel (every voxel once plus random repeats) as inds_reverse, height-band labels over 20 classes with 15 % set to the
ignore label 255, random colours; CPU tensors as the loader hands them over.  Network: MinkUNet18A / 34C with 20 classes,
eval mode, FusedMinkUNet(model).
  torch:   output = engine(coords.cuda(), feat.cuda()), output[inds_reverse], CrossEntropyLoss(ignore_index=255),
           max(1)[1], intersectionAndUnionGPU (three .cpu() histc and the .cpu().numpy() reads), the AverageMeter updates
           and loss.item(), as validate() does;
  device:  DeviceMinkValidation.add(coords, feat, inds_reverse, label) per scene, end() once after the last scene.
The arms alternate validation by validation on the same scenes.

Reported per architecture and arm (median over R validations): wall time per validation (host clock, ending in the result
on the host), the tail alone per scene (CUDA events: the torch arm after the forward, the device arm around its final
launch, osb_ce_head_eval), host synchronisations per scene made through torch (torch's sync debug mode, in a separate
untimed validation; the engine's own coordinate build is not counted in either arm), and both arms' (loss_avg, mIoU, mAcc,
allAcc).  Training: K (default 60) fused_train_step()s on 8 config1_50k scenes with SGD, the torch meters of train() (with
loss.item() and the .cpu() reads every step) against DeviceTrainMeter.add every step and read() every 10 steps
(print_freq), ms per step as the median of the two arms' alternating runs, and whether both gave the same per-step values.
Device name, power limit and the SM clock measured on the device between runs.  The JSON line is printed and, with --out,
written to DIR/bench_train_mink_validate.json."""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_distill_validate import AverageMeter, Events, intersection_and_union_gpu, make_scenes, power_limit_w  # noqa: E402

CLASSES = 20
IGNORE = 255


def torch_validation(eng, scenes, timing):
    criterion = torch.nn.CrossEntropyLoss(ignore_index=IGNORE)
    loss_meter, im, um, tm = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
    with torch.no_grad():
        for coords, feat, label, inds_reverse in scenes:
            timing.scene()
            label = label.cuda(non_blocking=True)
            output = eng(coords.cuda(non_blocking=True), feat.cuda(non_blocking=True))
            timing.tail_begin()
            output = output[inds_reverse, :]
            loss = criterion(output, label)
            output = output.detach().max(1)[1]
            intersection, union, target = intersection_and_union_gpu(output, label.detach(), CLASSES, IGNORE)
            intersection, union, target = intersection.cpu().numpy(), union.cpu().numpy(), target.cpu().numpy()
            im.update(intersection), um.update(union), tm.update(target)
            loss_meter.update(loss.item(), 1)
            timing.tail_end()
    timing.scene()
    iou_class = im.sum / (um.sum + 1e-10)
    accuracy_class = im.sum / (tm.sum + 1e-10)
    return loss_meter.avg, np.mean(iou_class), np.mean(accuracy_class), sum(im.sum) / (sum(tm.sum) + 1e-10)


def device_validation(eng, scenes, meter, timing):
    """the engine's tail hook wrapped so that the events (and the sync count) bracket the final launch only"""
    forward = type(eng)._forward

    def timed(coords, feats, cm, head, tail=None):
        def hooked(cur, n0, cm_):
            timing.tail_begin()
            r = tail(cur, n0, cm_)
            timing.tail_end()
            return r
        return forward(eng, coords, feats, cm, head, hooked if tail is not None else None)
    eng._forward = timed
    try:
        meter.begin()
        for coords, feat, label, inds_reverse in scenes:
            timing.scene()
            meter.add(coords, feat, inds_reverse, label)
        timing.scene()
        return meter.end(1)
    finally:
        del eng._forward


def count_syncs(fn):
    """torch synchronisations over a whole validation"""
    with warnings.catch_warnings(record=True) as log:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode(1)
        try:
            fn(Events())
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum('synchroniz' in str(w.message) for w in log)


def train_arms(dev, steps, print_freq=10):
    """train()'s step with the torch meters against DeviceTrainMeter, alternating runs of `steps` steps"""
    from bench_train_mink_step import labels_for
    from openscene_b200 import engine, synth, train_mink
    coords = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=i, batch_index=i)) for i in range(8)]).to(dev)
    labels = labels_for(coords.cpu(), CLASSES).to(dev)
    feats = torch.rand(coords.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(dev)
    model = synth.build_model('MinkUNet18A', CLASSES, seed=0).train().to(dev)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    snap_m = {k: v.clone() for k, v in model.state_dict().items()}

    def restore():
        with torch.no_grad():
            for k, v in model.state_dict().items():
                v.copy_(snap_m[k])
        opt.state.clear()

    def torch_meters():
        loss_meter, im, um, tm = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
        out = []
        for i in range(steps):
            torch.manual_seed(i)
            loss, pred = train_mink.fused_train_step(eng, opt, coords, feats, labels)
            intersection, union, target = intersection_and_union_gpu(pred, labels.detach().clone(), CLASSES, IGNORE)
            intersection, union, target = intersection.cpu().numpy(), union.cpu().numpy(), target.cpu().numpy()
            im.update(intersection), um.update(union), tm.update(target)
            accuracy = sum(im.val) / (sum(tm.val) + 1e-10)
            loss_meter.update(loss.item(), 8)
            out.append((loss_meter.val, accuracy, np.mean(intersection / (union + 1e-10)),
                        np.mean(intersection / (target + 1e-10))))
        return out

    def device_meter():
        meter = train_mink.DeviceTrainMeter(CLASSES)
        out = []
        for i in range(steps):
            torch.manual_seed(i)
            loss, pred = train_mink.fused_train_step(eng, opt, coords, feats, labels)
            meter.add(loss, pred, labels)
            if (i + 1) % print_freq == 0 or i + 1 == steps:
                out += [(s['loss'], s['accuracy'], s['mIoU'], s['mAcc']) for s in meter.read(weight=8)[0]]
        return out

    arms = {'torch_meters': torch_meters, 'device_train_meter': device_meter}
    rec = {k: [] for k in arms}
    vals = {}
    for rep in range(4):                                      # the first round warms up
        for name, fn in arms.items():
            restore()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            vals[name] = fn()
            torch.cuda.synchronize()
            if rep:
                rec[name].append((time.perf_counter() - t0) * 1e3 / steps)
    same = all(len(a) == len(b) and all(float(x) == float(y) for x, y in zip(a, b))
               for a, b in zip(vals['torch_meters'], vals['device_train_meter']))
    return {'steps_per_run': steps, 'voxels': coords.shape[0],
            'ms_per_step_median': {k: statistics.median(v) for k, v in rec.items()},
            'ms_per_step_all': rec, 'same_per_step_values': bool(same and len(vals['torch_meters']) == steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, default=16)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--archs', default='MinkUNet18A,MinkUNet34C')
    ap.add_argument('--train-steps', type=int, default=60)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from openscene_b200 import engine, synth, train_mink
    assert torch.cuda.is_available(), "bench_train_mink_validate.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    scenes = make_scenes(args.scenes)
    power = power_limit_w()
    sampler = ClockSampler(0, dev)
    result = {'metric': 'run/train_mink.py validate(): ms per validation, torch tail vs DeviceMinkValidation',
              'scenes': f"{args.scenes} scenes (config1_50k / config2_200k alternating), "
                        f"{sum(s[0].shape[0] for s in scenes)} voxels, {sum(len(s[3]) for s in scenes)} points, "
                        f"{CLASSES} classes",
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power, 'reps': args.reps, 'archs': {}}
    for arch in args.archs.split(','):
        model = synth.build_model(arch, CLASSES, seed=0).eval().to(dev)
        eng = engine.FusedMinkUNet(model)
        meter = train_mink.DeviceMinkValidation(eng, CLASSES)
        arms = {'torch_tail': lambda t: torch_validation(eng, scenes, t),
                'device_validation': lambda t: device_validation(eng, scenes, meter, t)}
        rec = {}
        for name, fn in arms.items():                        # warm-up, then the synchronisation count
            fn(Events())
            syncs = count_syncs(fn)
            torch.cuda.synchronize()
            rec[name] = {'host_syncs_per_scene': syncs / args.scenes, 'walls': [], 'tail': []}
        for _ in range(args.reps):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                sampler.sample()                             # stream-ordered, before the timed region
                torch.cuda.synchronize()
                t = Events()
                t0 = time.perf_counter()
                out = fn(t)
                torch.cuda.synchronize()
                rec[name]['walls'].append((time.perf_counter() - t0) * 1e3)
                _, tail = t.result()
                rec[name]['tail'].append(statistics.median(tail))
                rec[name]['result'] = [float(v) for v in out]
        for name in arms:
            r = rec[name]
            walls, tails = r.pop('walls'), r.pop('tail')
            r['ms_per_validation_median'] = statistics.median(walls)
            r['ms_per_validation_min_max'] = [min(walls), max(walls)]
            r['tail_ms_per_scene_median'] = statistics.median(tails)
        a, b = rec['torch_tail']['result'], rec['device_validation']['result']
        rec['same_metrics'] = a[1:] == b[1:]
        rec['loss_avg_difference'] = abs(a[0] - b[0])
        result['archs'][arch] = rec
        del eng, model, meter
        torch.cuda.empty_cache()
    sampler.sample()
    result['train'] = train_arms(dev, args.train_steps)
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_train_mink_validate.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
