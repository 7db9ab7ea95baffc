#!/usr/bin/env python
"""Test-time repeats of run/evaluate.py (``test_repeats > 1``, feature_type 'distill'): the reference's per-repeat host
round trip against ``repeat_eval.RepeatVote``.

    python scripts/bench_repeat_eval.py [--scenes S] [--repeats R] [--k 20 80] [--scene config1_50k] [--out DIR]

Workload: S synthetic scenes (``synth.scene_points(name, seed=i)``) x R repeats.  Every repeat re-voxelises every scene on
the device (``voxelize_points``) with a fresh random rotation / scale (the evaluation voxeliser's augmentation) and runs
MinkUNet18A with a 768-d head on ``FusedMinkUNet``.  The same network output then goes through both tails, the order of
the two alternating from scene to scene:

  reference  ``pred = predictions[inds_reverse].half() @ text.t()``; ``preds.append(pred.cpu())``; at the end of the
             repeat on the host: ``torch.cat``, ``store = pred + store``, ``.float().max(1)[1]`` of both and the metric
             (``oracle.metric_ref``, the restatement of util/metric.py) for the current and the accumulated labels
  device     ``RepeatVote.match_distill`` per scene (vote fused into the match epilogue, confusion matrices on the device);
             ``end_repeat()`` at the end of the repeat

Reported per K and per repeat: the post-network time per scene (CUDA events around the tail, median over scenes; for the
reference it includes the synchronous ``.cpu()``), the end-of-repeat host wall time, both IoUs of both arms and the
agreement of the accumulated labels.  Fields ending in ``_from_shapes`` are computed from the tensor shapes, not measured:
the bytes copied device to host and the host memory the score matrices hold at the peak of the reference's end-of-repeat
(the per-scene list, its concatenation, the store and the ``.float()`` temporary).  Per K also the time per launch of the
match kernel alone on the last scene: labels only, with the fp16 scores written, and with the vote epilogue.  Also the
device name, power limit and SM clocks.  The JSON line is printed and, with --out, written to DIR/bench_repeat_eval.json."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def scene_labels(pts, k):
    """ground truth from the geometry: height bands x slabs, 5 % unlabelled (255)"""
    p = torch.from_numpy(pts)
    lab = ((p[:, 2] * 5).long() * 3 + (p[:, 0] * 4).long()) % k
    lab[torch.arange(len(p)) % 20 == 0] = 255
    return lab


def run(k, args, eng, scenes, gts_host, gts_dev, dev, sampler):
    from oracle import metric_ref
    from openscene_b200 import synth
    from openscene_b200.repeat_eval import RepeatVote
    from openscene_b200.voxelize import Voxelizer, voxelize_points
    text = torch.from_numpy(synth.text_embeddings(k, 768)).to(dev)
    vox = Voxelizer(voxel_size=scenes[0][1], use_augmentation=True, scale_augmentation_bound=(0.9, 1.1),
                    rotation_augmentation_bound=((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi)))
    np.random.seed(0)
    gt_all = torch.cat(gts_host).numpy()
    n_all = len(gt_all)
    vote = RepeatVote(k)
    store = 0.0
    reps = []
    for r in range(args.repeats + 1):                 # repeat 0 is a warm-up of both tails on a throw-away vote
        warm = r == 0
        if warm:
            v = RepeatVote(k)
            v.begin_repeat()
        else:
            vote.begin_repeat()
            v = vote
        preds, t_ref, t_dev = [], [], []
        d2h = 0
        for s, (pts, _) in enumerate(scenes):
            M_v, M_r = vox.get_transformation_matrix()
            cv, inds, inv, _ = voxelize_points(torch.from_numpy(pts).to(dev), M_r @ M_v)
            c4 = torch.zeros((cv.shape[0], 4), dtype=torch.int32, device=dev)
            c4[:, 1:] = cv
            with torch.no_grad():
                out = eng(c4, torch.ones(cv.shape[0], 3, device=dev))

            def ref_tail():
                pred = out[inv].half() @ text.t()
                preds.append(pred.cpu())

            def dev_tail():
                v.match_distill(s, out, inv, text, gt=gts_dev[s])
            order = (('ref', ref_tail), ('dev', dev_tail)) if s % 2 == 0 else (('dev', dev_tail), ('ref', ref_tail))
            for name, fn in order:
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); fn(); b.record()
                b.synchronize()
                (t_ref if name == 'ref' else t_dev).append(a.elapsed_time(b))
            d2h += preds[-1].numel() * 2
        if warm:
            v.end_repeat()
            continue
        t0 = time.perf_counter()
        pred = torch.cat(preds)
        cur = pred.float().max(1)[1]
        store = pred + store
        acc = store.float().max(1)[1]
        iou_ref = (metric_ref.mean_iou(cur.numpy(), gt_all, k)[0], metric_ref.mean_iou(acc.numpy(), gt_all, k)[0])
        host_ref = time.perf_counter() - t0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        iou_dev = vote.end_repeat()
        host_dev = time.perf_counter() - t0
        lab = vote.labels().cpu()
        agree = float((lab == acc).float().mean())
        n_bytes = n_all * k * 2
        reps.append({
            'repeat': r - 1, 'points': n_all,
            'tail_ms_per_scene_median': {'reference': statistics.median(t_ref), 'device': statistics.median(t_dev)},
            'tail_ms_sum': {'reference': sum(t_ref), 'device': sum(t_dev)},
            'end_of_repeat_host_ms': {'reference': 1e3 * host_ref, 'device': 1e3 * host_dev},
            # computed from shapes, not measured: the reference copies every scene's fp16 scores; end_repeat copies the
            # [C,C] confusion block, the C ground-truth counts and the int32 bad-label count of each of its two meters
            'd2h_bytes_from_shapes': {'reference': d2h, 'device': 2 * ((k * k + k) * 8 + 4)},
            # computed from shapes: the per-scene list, its concatenation, the store and the .float() temporary
            'host_score_bytes_peak_from_shapes': {'reference': n_bytes * 3 + n_all * k * 4, 'device': 0},
            'device_store_bytes_from_shapes': n_bytes,
            'iou_current': {'reference': iou_ref[0], 'device': iou_dev[0]},
            'iou_accumulated': {'reference': iou_ref[1], 'device': iou_dev[1]},
            'accumulated_label_agreement': agree})
        del preds, pred
        sampler.sample()
    kt = kernel_times(out, inv, text, dev)
    return {'repeats': reps, 'match_kernel_ms_last_scene': kt}


def kernel_times(feat, inv, text, dev, reps=30, rounds=5):
    """CUDA-event time per launch on one scene: the tensor-core match writing labels only, the same writing the fp16
    scores too, and the match with the vote epilogue (store read + written, two labels).  Arms alternate per round."""
    from openscene_b200 import _cabi as C
    n_vox, c = feat.shape
    n_pts, k = inv.shape[0], text.shape[0]
    scores = torch.empty((n_pts, k), dtype=torch.float16, device=dev)
    lab = torch.empty(n_pts, dtype=torch.int64, device=dev)
    lab2 = torch.empty(n_pts, dtype=torch.int64, device=dev)
    store = torch.zeros((n_pts, k), dtype=torch.float16, device=dev)
    s = C.stream_ptr()
    arms = {
        'match_labels': lambda: C.call('osb_match_scores', C.ptr(feat), 0, n_vox, c, C.ptr(inv), n_pts, C.ptr(text), k, 0,
                                       None, C.ptr(lab), None, s),
        'match_scores_and_labels': lambda: C.call('osb_match_scores', C.ptr(feat), 0, n_vox, c, C.ptr(inv), n_pts,
                                                  C.ptr(text), k, 0, C.ptr(scores), C.ptr(lab), None, s),
        'match_vote': lambda: C.call('osb_match_vote', C.ptr(feat), 0, n_vox, c, C.ptr(inv), n_pts, C.ptr(text), k, 0, None,
                                     C.ptr(store), C.ptr(lab), C.ptr(lab2), s)}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {n: [] for n in arms}
    for _ in range(rounds):
        for n, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            b.synchronize()
            times[n].append(a.elapsed_time(b) / reps)
    return {'points': n_pts, 'voxels': n_vox, 'k': k,
            **{n: {'ms_min': min(t), 'ms_median': statistics.median(t)} for n, t in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, default=16)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--k', type=int, nargs='+', default=[20, 80])
    ap.add_argument('--scene', default='config1_50k')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    from bench import ClockSampler
    from bench_batch_stats import power_limit_w
    from openscene_b200 import engine, synth
    assert torch.cuda.is_available(), "bench_repeat_eval.py needs a CUDA device (no CPU fallback)"
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    scenes = [synth.scene_points(args.scene, seed=i) for i in range(args.scenes)]
    power_w, power_how = power_limit_w(0)
    sampler = ClockSampler(0, dev)
    model = synth.build_model('MinkUNet18A', 768, seed=0).eval().to(dev)
    eng = engine.FusedMinkUNet(model)
    result = {'metric': 'test-time repeat tail of run/evaluate.py: host round trip vs device vote',
              'workload': f'{args.scenes} x {args.scene}, {args.repeats} repeats, MinkUNet18A 768-d on FusedMinkUNet, '
                          f'feature_type distill',
              'device': torch.cuda.get_device_name(dev), 'power_limit_w': power_w, 'power_limit_source': power_how,
              'runs': {}}
    for k in args.k:
        gts_host = [scene_labels(p, k) for p, _ in scenes]
        gts_dev = [g.to(dev) for g in gts_host]
        result['runs'][f'K={k}'] = run(k, args, eng, scenes, gts_host, gts_dev, dev, sampler)
    result['clocks'] = sampler.stop()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_repeat_eval.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
