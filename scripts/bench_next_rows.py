"""Measure the SURVEY 8f 'next' rows on the GPU: multi-view fusion accumulate and the segmentation metrics.
Prints one JSON line per row (CUDA-event timed, warm, inputs resident in HBM) with the HBM roofline fraction and a
CPU-oracle baseline on a bounded sample.  Not part of bench.py's contract (that is the north-star path)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openscene_b200 import _cabi as C                                 # noqa: E402
from openscene_b200.fusion import FeatureFusion, PointCloudToImageMapper   # noqa: E402
from openscene_b200 import metric                                     # noqa: E402
from openscene_b200.synth import fusion_case                          # noqa: E402


def peak_gbs():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        return float(json.load(open(p))['hbm_gbs']), 'measured (MEASURED_PEAKS.json)'
    return 3350.0, 'data sheet (H100 SXM HBM3, 700 W card), not measured'


def timed(fn, reps=10, warm=3):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for _ in range(warm):
        fn()
    ms = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def bench_fusion(n=1_000_000, c=768, F=32):
    from oracle import fusion_ref
    pts, poses, depths, intr = fusion_case(77, n, True, n_frames=F)
    mapper = PointCloudToImageMapper(image_dim=(320, 240), intrinsics=intr, cut_bound=10, device='cuda')
    feats = (torch.randn(F, 240, 320, c, device='cuda') * 0.5).half()
    fuser = FeatureFusion(pts, c, mapper)
    d_dev = torch.stack([torch.from_numpy(d) for d in depths]).cuda()
    l0 = C.lib().osb_launch_count()
    fuser.add_frames(poses, list(d_dev), feats)
    launches = C.lib().osb_launch_count() - l0
    ms = timed(lambda: fuser.add_frames(poses, list(d_dev), feats))
    maps = torch.stack([mapper.compute_mapping(p, pts, d, as_tensor=True) for p, d in zip(poses, depths)])
    vis = maps[:, :, 2].long()
    pairs, touched = int(vis.sum()), int((vis.sum(0) > 0).sum())
    # algorithmic bytes: points once per frame (24 B), depth probe (8 B) per in-image pair ~ per pair, the pixel feature
    # (2C) per visible pair, the fp32 sum row read + written once per touched point (8C), counter (8 B)
    alg = 24 * n + 8 * pairs + 2 * c * pairs + 8 * c * touched + 8 * touched
    peak, src = peak_gbs()
    # CPU oracle on a bounded sample: 4 frames, 100k points
    ns, Fs = 100_000, 4
    t0 = time.time()
    fusion_ref.fuse_frames(pts[:ns], poses[:Fs], depths[:Fs], [f.cpu() for f in feats[:Fs]], intr, (320, 240), 10)
    cpu_s = time.time() - t0
    print(json.dumps({'row': '8f-2 fusion accumulate', 'points': n, 'frames_per_call': F, 'feat_dim': c, 'ms_per_call': ms,
                      'point_frames_per_s': n * F / ms * 1e3, 'visible_pairs': pairs, 'touched_points': touched,
                      'gpu_launches_per_call': int(launches),
                      'roofline': {'bound': 'hbm', 'achieved': alg / ms / 1e6, 'peak': peak, 'unit': 'GB/s', 'frac': alg / ms / 1e6 / peak,
                                   'peak_source': src, 'algorithmic_bytes': alg},
                      'cpu_baseline': {'value': ns * Fs / cpu_s, 'unit': 'point-frames/s', 'cores': torch.get_num_threads(), 'kind': 'port',
                                       'sample': f'{ns} points x {Fs} frames, {cpu_s:.1f} s'}}))


def bench_metric(n=20_000_000, Cn=20):
    from oracle import metric_ref
    g = torch.Generator(device='cuda').manual_seed(0)
    gt = torch.randint(0, Cn, (n,), device='cuda', generator=g)
    gt[torch.rand(n, device='cuda', generator=g) < 0.1] = 255
    pred = torch.where(torch.rand(n, device='cuda', generator=g) < 0.6, gt.clamp(max=Cn - 1), torch.randint(0, Cn, (n,), device='cuda', generator=g))
    meter = metric.ConfusionMeter(Cn)
    ms = timed(lambda: meter.update(pred, gt))
    ms_iu = timed(lambda: metric.intersectionAndUnionGPU(pred, gt, Cn, 255))
    peak, src = peak_gbs()
    alg = 16 * n
    ns = 2_000_000
    p, q = pred[:ns].cpu().numpy(), gt[:ns].cpu().numpy()
    t0 = time.time(); metric_ref.confusion_matrix(p, q, Cn); cpu_s = time.time() - t0
    print(json.dumps({'row': '8f-4 confusion matrix / intersection-union', 'labels': n, 'classes': Cn, 'dtype': 'int64',
                      'confusion_ms': ms, 'inter_union_ms': ms_iu, 'labels_per_s': n / ms * 1e3,
                      'roofline': {'bound': 'hbm', 'achieved': alg / ms / 1e6, 'peak': peak, 'unit': 'GB/s', 'frac': alg / ms / 1e6 / peak,
                                   'peak_source': src, 'algorithmic_bytes': alg},
                      'cpu_baseline': {'value': ns / cpu_s, 'unit': 'labels/s', 'cores': 1, 'kind': 'port', 'sample': f'{ns} labels, {cpu_s:.2f} s'}}))


def bench_voxelize(scene='config2_200k'):
    """SURVEY 8f-1 / a1-a2: float points -> voxel coords, inds, inds_reverse (csrc/voxelize.cu: k_vox_*, radix sort, unique)."""
    from openscene_b200 import synth
    from openscene_b200.voxelize import voxelize_points
    from oracle import voxelize_ref
    pts_np, vsz = synth.scene_points(scene, 0)
    pts = torch.from_numpy(pts_np).cuda()
    mat = np.eye(4); np.fill_diagonal(mat[:3, :3], 1.0 / vsz)
    n_pts = len(pts_np)
    l0 = C.lib().osb_launch_count()
    cv, inds, inv, _ = voxelize_points(pts, mat)
    launches = C.lib().osb_launch_count() - l0
    n_vox = cv.shape[0]
    ms = timed(lambda: voxelize_points(pts, mat))
    alg = 3 * pts.element_size() * n_pts + 8 * n_pts + 8 * n_vox + 12 * n_vox    # points in; inds_reverse, inds and the voxel coords out
    peak, src = peak_gbs()
    ns = min(n_pts, 200_000)
    t0 = time.time(); voxelize_ref.voxelize(pts_np[:ns], mat); cpu_s = time.time() - t0
    print(json.dumps({'row': '8f-1 voxeliser (k_vox_* + radix sort + unique)', 'scene': scene, 'points': n_pts, 'voxels': int(n_vox), 'ms_per_call': ms,
                      'points_per_s': n_pts / ms * 1e3, 'gpu_launches_per_call': int(launches),
                      'roofline': {'bound': 'hbm', 'achieved': alg / ms / 1e6, 'peak': peak, 'unit': 'GB/s', 'frac': alg / ms / 1e6 / peak,
                                   'peak_source': src, 'algorithmic_bytes': alg,
                                   'note': 'algorithmic bytes count the inputs and outputs once; the 8-pass LSD radix sort of 64-bit keys + '
                                           '32-bit payloads alone moves 8 x 24 B per point, so the kernel sequence is launch- and pass-bound at this size'},
                      'cpu_baseline': {'value': ns / cpu_s, 'unit': 'points/s', 'cores': 1, 'kind': 'port', 'sample': f'{ns} points, {cpu_s:.2f} s'}}))


def bench_remap(n_pts=2_000_000, c=768):
    """SURVEY 8f-3 loader-side remap (csrc/remap.cu: k_remap_*): per-voxel feature mask + gathered fp16 feature rows."""
    from openscene_b200.fused_features import remap_fused_features
    g = torch.Generator(device='cuda').manual_seed(0)
    mask_full = torch.rand(n_pts, device='cuda', generator=g) < 0.6
    m_rows = int(mask_full.sum())
    feat = (torch.randn(m_rows, c, device='cuda', generator=g) * 0.3).half()
    n_vox = n_pts * 2 // 5
    vox_ind = torch.sort(torch.randperm(n_pts, device='cuda', generator=g)[:n_vox])[0]
    out = {}
    for split in ('train', 'val'):
        f, m = remap_fused_features(feat, mask_full, vox_ind, split)
        kept = int(m.sum())
        ms = timed(lambda: remap_fused_features(feat, mask_full, vox_ind, split))
        rows_written = kept if split == 'train' else n_vox
        alg = n_pts + 8 * n_vox + 2 * c * kept + 2 * c * rows_written + n_vox
        peak, src = peak_gbs()
        out[split] = {'ms_per_call': ms, 'kept_voxels': kept, 'rows_written': rows_written,
                      'roofline': {'bound': 'hbm', 'achieved': alg / ms / 1e6, 'peak': peak, 'unit': 'GB/s', 'frac': alg / ms / 1e6 / peak,
                                   'peak_source': src, 'algorithmic_bytes': alg}}
    print(json.dumps({'row': '8f-3 fused-feature remap (k_remap_*)', 'points': n_pts, 'voxels': n_vox, 'feature_rows': m_rows, 'feat_dim': c,
                      'note': 'time includes the wrapper (mask cast, output allocation) around osb_feature_remap', **out}))


def bench_container(n_pts=1_000_000, c=768):
    """SURVEY 8f-3 container: file (page cache) -> device, remap fused into the read, against torch.load of the reference's
    pickle + the loader-side remap kernel."""
    import tempfile
    from openscene_b200 import fused_container as fc
    from openscene_b200.fused_features import remap_fused_features
    g = torch.Generator().manual_seed(0)
    mask_full = torch.rand(n_pts, generator=g) < 0.6
    feat = (torch.randn(int(mask_full.sum()), c, generator=g) * 0.3).half()
    vox_ind = torch.randperm(n_pts, generator=g)[:n_pts * 2 // 5]
    with tempfile.TemporaryDirectory() as td:
        pt, ob = os.path.join(td, 's.pt'), os.path.join(td, 's.osbf')
        torch.save({'feat': feat, 'mask_full': mask_full}, pt)
        fc.convert_torch_save(pt, ob)
        f = fc.FusedFeatureFile(ob)

        def wall(fn, reps=5):
            fn(); ts = []
            for _ in range(reps):
                torch.cuda.synchronize(); t0 = time.time(); fn(); torch.cuda.synchronize(); ts.append(time.time() - t0)
            return float(np.median(ts)) * 1e3

        def via_pickle():
            d = torch.load(pt, map_location='cpu', weights_only=False)
            return remap_fused_features(d['feat'], d['mask_full'], vox_ind, 'train')
        ms_c = wall(lambda: f.read_remapped(vox_ind, 'train', 'cuda'))
        ms_p = wall(via_pickle)
        kept = int(f.rows_for(vox_ind.numpy())[1].sum())
        print(json.dumps({'row': '8f-3 fused-feature container', 'points': n_pts, 'feature_rows': int(feat.shape[0]), 'feat_dim': c,
                          'voxels': int(vox_ind.numel()), 'kept_rows': kept, 'file_bytes': os.path.getsize(ob),
                          'container_ms': ms_c, 'container_GBps_of_kept_rows': kept * c * 2 / ms_c / 1e6,
                          'torch_load_plus_remap_ms': ms_p, 'speedup': ms_p / ms_c,
                          'note': 'wall clock, file in the page cache; container: bitmap rank query + gather of the kept rows from the mapping '
                                  'into pinned memory + async H2D; baseline: torch.load of the whole pickle, H2D of all rows, osb_feature_remap'}))


if __name__ == '__main__':
    which = sys.argv[1:] or ['fusion', 'metric', 'voxelize', 'remap', 'container']
    if 'fusion' in which: bench_fusion()
    if 'metric' in which: bench_metric()
    if 'voxelize' in which:
        bench_voxelize('config2_200k')
        bench_voxelize('config5_lidar')
    if 'remap' in which: bench_remap()
    if 'container' in which: bench_container()
