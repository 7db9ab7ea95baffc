#!/usr/bin/env python
"""One run/distill.py validation (validate(), :403-447) with the batch-statistics engine forward in both arms: the
reference's torch tail after the forward against openscene_b200.distill.DeviceValidation.

    python scripts/bench_distill_validate.py [--scenes N] [--reps R] [--archs A,B] [--out DIR]

Scenes: N (default 16) synthetic rooms, half synth.scene('config1_50k', seed=i) and half 'config2_200k', each with
1.5 points per voxel (every voxel once plus random repeats) as inds_reverse, height-band labels over 20 classes with 15 %
set to the ignore label 255, random colours; CPU tensors as the loader hands them over.  Text: 20 unit fp16 embeddings.
Per scene both arms run ``engine(coords.cuda(), feat.cuda())`` (FusedMinkUNet(model, batch_stats=True)), then
  torch:   output[inds_reverse].half() @ text.t(), CrossEntropyLoss(ignore_index=255), max(1)[1], intersectionAndUnionGPU
           (three .cpu() histc and the .cpu().numpy() reads), the AverageMeter updates and loss.item(), as validate() does;
  device:  DeviceValidation.add(output, inds_reverse, label); end() once after the last scene.
The arms alternate validation by validation on the same scenes.

Reported per architecture and arm (median over R validations): wall time per validation (host clock, ending in the result
on the host), the median scene time (CUDA events at scene boundaries), the tail alone (CUDA events around the tail of
each scene: median per scene and sum per validation), host synchronisations per scene in the tail (torch's sync debug mode,
in a separate untimed validation), and both arms' (loss_avg, mIoU, mAcc, allAcc).  The torch arm's scores come from
cuBLAS, the device arm's from the tensor-core match, so argmax near-ties may differ between them.  Device name, power
limit (read before the timed region) and the SM clock measured on the device between validations (osb_measure_sm_mhz;
no NVML query inside a timed region).  The JSON line is printed and, with --out, written to DIR/bench_distill_validate.json."""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

CLASSES = 20
IGNORE = 255


class AverageMeter:
    """util/util.py:86-102."""

    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def intersection_and_union_gpu(output, target, K, ignore_index=IGNORE):
    """util/util.py:132-145."""
    output = output.view(-1)
    target = target.view(-1)
    output[target == ignore_index] = ignore_index
    intersection = output[output == target]
    area_intersection = torch.histc(intersection.float().cpu(), bins=K, min=0, max=K - 1)
    area_output = torch.histc(output.float().cpu(), bins=K, min=0, max=K - 1)
    area_target = torch.histc(target.float().cpu(), bins=K, min=0, max=K - 1)
    area_union = area_output + area_target - area_intersection
    return area_intersection.cuda(), area_union.cuda(), area_target.cuda()


def make_scenes(n):
    from openscene_b200 import synth
    out = []
    for i in range(n):
        name = 'config1_50k' if i % 2 == 0 else 'config2_200k'
        coords = torch.from_numpy(synth.scene(name, seed=i // 2))
        g = torch.Generator().manual_seed(i)
        n_vox = coords.shape[0]
        inv = torch.cat([torch.randperm(n_vox, generator=g), torch.randint(0, n_vox, (n_vox // 2,), generator=g)])
        z = coords[:, 3].float()
        label = (z / (z.max() + 1) * CLASSES).long()[inv]
        label[torch.rand(len(inv), generator=g) < 0.15] = IGNORE
        out.append((coords, torch.rand(n_vox, 3, generator=g), label, inv))
    return out


def torch_validation(eng, scenes, text, timing):
    criterion = torch.nn.CrossEntropyLoss(ignore_index=IGNORE)
    loss_meter, im, um, tm = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
    with torch.no_grad():
        for coords, feat, label, inds_reverse in scenes:
            timing.scene()
            output = eng(coords.cuda(non_blocking=True), feat.cuda(non_blocking=True))
            label = label.cuda(non_blocking=True)
            timing.tail_begin()
            output = output[inds_reverse, :]
            output = output.half() @ text.t()
            loss = criterion(output, label)
            output = torch.max(output, 1)[1]
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
    meter.begin()
    with torch.no_grad():
        for coords, feat, label, inds_reverse in scenes:
            timing.scene()
            output = eng(coords.cuda(non_blocking=True), feat.cuda(non_blocking=True))
            timing.tail_begin()
            meter.add(output, inds_reverse, label)
            timing.tail_end()
    timing.scene()
    return meter.end(1)


class Events:
    """CUDA events at scene boundaries and around each tail; with ``syncs``, the tail runs under torch's sync debug mode
    and its synchronisations are counted."""

    def __init__(self, syncs=False):
        self.bounds, self.tails, self.syncs, self.count = [], [], syncs, 0
        self._rec = None

    def _ev(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def scene(self):
        self.bounds.append(self._ev())

    def tail_begin(self):
        if self.syncs:
            self._rec = warnings.catch_warnings(record=True)
            self._log = self._rec.__enter__()
            warnings.simplefilter('always')
            torch.cuda.set_sync_debug_mode(1)
        self.tails.append([self._ev()])

    def tail_end(self):
        self.tails[-1].append(self._ev())
        if self.syncs:
            torch.cuda.set_sync_debug_mode(0)
            self.count += sum('synchroniz' in str(w.message) for w in self._log)
            self._rec.__exit__(None, None, None)

    def result(self):
        scene = [a.elapsed_time(b) for a, b in zip(self.bounds[:-1], self.bounds[1:])]
        tail = [a.elapsed_time(b) for a, b in self.tails]
        return scene, tail


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:                                        # noqa: BLE001
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, default=16)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--archs', default='MinkUNet18A,MinkUNet34C')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from openscene_b200 import distill, engine, synth
    assert torch.cuda.is_available(), "bench_distill_validate.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    scenes = make_scenes(args.scenes)
    text = torch.from_numpy(synth.text_embeddings(CLASSES)).to(dev)
    power = power_limit_w()
    sampler = ClockSampler(0, dev)
    result = {'metric': 'run/distill.py validate(): ms per validation, torch tail vs DeviceValidation',
              'scenes': f"{args.scenes} scenes (config1_50k / config2_200k alternating), "
                        f"{sum(s[0].shape[0] for s in scenes)} voxels, {sum(len(s[3]) for s in scenes)} points, "
                        f"{CLASSES} classes",
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power, 'reps': args.reps, 'archs': {}}
    for arch in args.archs.split(','):
        model = synth.build_model(arch, 768, seed=0).train().to(dev)
        eng = engine.FusedMinkUNet(model, batch_stats=True)
        meter = distill.DeviceValidation(text, CLASSES)
        arms = {'torch_tail': lambda t: torch_validation(eng, scenes, text, t),
                'device_validation': lambda t: device_validation(eng, scenes, meter, t)}
        rec = {}
        for name, fn in arms.items():                        # warm-up, then the synchronisation count
            fn(Events())
            t = Events(syncs=True)
            fn(t)
            torch.cuda.synchronize()
            rec[name] = {'host_syncs_per_scene_in_tail': t.count / args.scenes, 'walls': [], 'scene': [], 'tail': []}
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
                scene, tail = t.result()
                rec[name]['scene'].append(statistics.median(scene))
                rec[name]['tail'].append((statistics.median(tail), sum(tail)))
                rec[name]['result'] = [float(v) for v in out]
        for name in arms:
            r = rec[name]
            walls, tails = r.pop('walls'), r.pop('tail')
            r['ms_per_validation_median'] = statistics.median(walls)
            r['ms_per_validation_min_max'] = [min(walls), max(walls)]
            r['ms_per_scene_median'] = statistics.median(r.pop('scene'))
            r['tail_ms_per_scene_median'] = statistics.median(t[0] for t in tails)
            r['tail_ms_per_validation_median'] = statistics.median(t[1] for t in tails)
        result['archs'][arch] = rec
        del eng, model, meter
        torch.cuda.empty_cache()
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_distill_validate.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
