"""Generate tests/golden/*.npz in the build container (needs /root/reference; NOT run on the GPU box).

1. voxelizer_*.npz : outputs of the reference's own ``dataset/voxelizer.py`` (imported unmodified, with the
   ``collections.Sequence/Iterable`` aliases Python 3.12 needs) for seeded inputs + the exact 4x4 matrix it drew.
2. unet_*.npz      : activations of the reference's unmodified ``models/mink_unet.py`` run on the CPU oracle
   (oracle/me_cpu.py registered as ``MinkowskiEngine``) in fp64, seeded weights, eval-mode BN with randomised
   statistics, on a small synthetic room.  These pin the *topology*; the ME arithmetic itself is the oracle's
   (parity unpinned against real MinkowskiEngine -- see oracle/__init__.py).

3. fusion_mapping_*.npz : outputs of the reference's own ``PointCloudToImageMapper.compute_mapping``
   (scripts/feature_fusion/fusion_util.py, imported with a stub ``tensorflow`` the method never touches) for seeded
   points, camera poses and z-buffer depth images.
4. metric_*.npz    : outputs of the reference's ``util/metric.py`` and ``util/util.py`` intersection/union helpers
   (stub ``open3d`` / ``clip`` / ``matplotlib``; ``Tensor.cuda`` patched to the identity -- no GPU here).

5. loader_*.npz    : what the reference's own ``FusedFeatureLoader.__getitem__`` (dataset/feature_loader.py) returns for
   synthetic scene / fused-feature files written to a scratch directory (``SharedArray`` stubbed; ``torch.load`` given
   the ``weights_only=False`` default of the PyTorch the reference targets), plus the 4x4 matrix its voxeliser drew.

6. augment_*.npz   : the reference's own ``dataset/augmentation.py`` transforms and the ``aug=True`` items of its
   ``Point3DLoader`` / ``FusedFeatureLoader`` (same stubs as 5.) for seeded inputs.  Each case stores its inputs, the
   seed of both global generators, the outputs and the next draws of ``random`` and ``np.random`` after the call.

Usage: python scripts/make_golden.py [voxelizer] [unet] [fusion] [metric] [loader] [augment]
"""
import collections
import collections.abc
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference'
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, 'tests', 'golden')


def golden_voxelizer():
    collections.Sequence = collections.abc.Sequence      # voxelization_utils.py:6
    collections.Iterable = collections.abc.Iterable      # voxelizer.py:55
    sys.path.insert(0, REF)
    from dataset.voxelizer import Voxelizer
    cases = {
        'aug_f64': dict(n=4000, extent=3.0, voxel=0.05, aug=True, dtype=np.float64, seed=1),
        'noaug_f32': dict(n=3000, extent=2.0, voxel=0.05, aug=False, dtype=np.float32, seed=2),
        'dups_f64': dict(n=5000, extent=0.6, voxel=0.05, aug=True, dtype=np.float64, seed=3),
        'neg_f64': dict(n=2000, extent=4.0, voxel=0.02, aug=True, dtype=np.float64, seed=4, shift=-2.0),
    }
    for name, c in cases.items():
        rng = np.random.RandomState(c['seed'])
        pts = (rng.rand(c['n'], 3) * c['extent'] + c.get('shift', 0.0)).astype(c['dtype'])
        vox = Voxelizer(voxel_size=c['voxel'], clip_bound=None, use_augmentation=c['aug'],
                        scale_augmentation_bound=(0.9, 1.1),
                        rotation_augmentation_bound=((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi)),
                        translation_augmentation_ratio_bound=((-0.2, 0.2), (-0.2, 0.2), (0, 0)))
        np.random.seed(c['seed'] + 100)
        M_v, M_r = vox.get_transformation_matrix()
        rigid = (M_r @ M_v) if c['aug'] else M_v
        np.random.seed(c['seed'] + 100)          # same draws inside voxelize()
        feats = np.zeros((c['n'], 3), dtype=np.float32)
        labels = np.zeros(c['n'], dtype=np.int64)
        coords_aug, _, _, inds_rec, inds = vox.voxelize(pts, feats, labels, return_ind=True)
        np.savez_compressed(os.path.join(OUT, f'voxelizer_{name}.npz'), points=pts, matrix=rigid,
                            coords_vox=coords_aug, inds=np.asarray(inds), inds_reverse=np.asarray(inds_rec))
        print(name, 'points', c['n'], '-> voxels', len(inds))


def golden_unet():
    from oracle import me_cpu
    me_cpu.install_as_minkowski_engine()
    sys.path.insert(0, REF)
    from models.mink_unet import mink_unet as ref_mink_unet
    from openscene_b200 import synth
    coords = synth.scene('tiny')
    print('tiny scene voxels', len(coords))
    for arch in ('MinkUNet18A', 'MinkUNet34C'):
        torch.manual_seed(0)
        model = ref_mink_unet(in_channels=3, out_channels=768, D=3, arch=arch)
        synth.randomize_bn_stats(model, 1)
        model = model.double().eval()
        rng = np.random.RandomState(7)
        feats = torch.from_numpy(rng.rand(len(coords), 3).astype(np.float32)).double()   # fp32-representable
        with torch.no_grad():
            x = me_cpu.SparseTensor(feats, torch.from_numpy(coords))
            out = model(x)
        out = out.numpy()
        rows = np.sort(np.random.RandomState(11).choice(len(coords), 128, replace=False))
        keys = list(model.state_dict().keys())
        shapes = [tuple(v.shape) for v in model.state_dict().values()]
        np.savez_compressed(os.path.join(OUT, f'unet_{arch}.npz'), coords=coords, feats=feats.numpy().astype(np.float32),
                            rows=rows, out_rows=out[rows].astype(np.float32),
                            row_norm=np.linalg.norm(out, axis=1).astype(np.float32),
                            col_sum=out.sum(0).astype(np.float64),
                            state_keys=np.array(keys), state_shapes=np.array([str(s) for s in shapes]),
                            n_params=np.int64(sum(p.numel() for p in model.parameters())))
        print(arch, 'params', sum(p.numel() for p in model.parameters()), 'out', out.shape, 'abs mean', np.abs(out).mean())


def _stub_modules(*names):
    import types
    for nm in names:
        parts = nm.split('.')
        for i in range(1, len(parts) + 1):
            sub = '.'.join(parts[:i])
            if sub not in sys.modules:
                sys.modules[sub] = types.ModuleType(sub)
            if i > 1:
                setattr(sys.modules['.'.join(parts[:i - 1])], parts[i - 1], sys.modules[sub])


def golden_fusion():
    _stub_modules('tensorflow', 'tensorflow.io', 'tensorflow.compat', 'tensorflow.compat.v1')
    sys.path.insert(0, os.path.join(REF, 'scripts', 'feature_fusion'))
    from fusion_util import PointCloudToImageMapper, adjust_intrinsic, make_intrinsic
    from openscene_b200.synth import fusion_case
    # the intrinsics helpers with the ScanNet / Matterport-style numbers the fusion scripts use (scannet_openseg.py:124-160)
    k0 = make_intrinsic(fx=577.870605, fy=577.870605, mx=319.5, my=239.5)
    k1 = adjust_intrinsic(k0.copy(), intrinsic_image_dim=[640, 480], image_dim=(320, 240))
    k2 = adjust_intrinsic(make_intrinsic(1075.1, 1075.8, 629.7, 522.3), intrinsic_image_dim=[1280, 1024], image_dim=(640, 512))
    np.savez_compressed(os.path.join(OUT, 'fusion_intrinsics.npz'), k0=k0, k1=k1, k2=k2)
    cases = {'depth_cut10': dict(seed=21, n=6000, with_depth=True, cut=10),
             'depth_cut0': dict(seed=22, n=5000, with_depth=True, cut=0),
             'nodepth_cut5': dict(seed=23, n=5000, with_depth=False, cut=5)}
    for name, c in cases.items():
        pts, poses, depths, intr = fusion_case(c['seed'], c['n'], c['with_depth'])
        mapper = PointCloudToImageMapper(image_dim=(320, 240), intrinsics=intr, visibility_threshold=0.25, cut_bound=c['cut'])
        maps = np.stack([mapper.compute_mapping(p, pts, d) for p, d in zip(poses, depths)])
        np.savez_compressed(os.path.join(OUT, f'fusion_mapping_{name}.npz'), seed=c['seed'], n=c['n'], with_depth=c['with_depth'],
                            cut=c['cut'], mapping=maps.astype(np.int32))
        print('fusion', name, 'visible per frame', maps[:, :, 2].sum(1))


def golden_metric():
    _stub_modules('open3d', 'clip', 'matplotlib', 'matplotlib.patches', 'matplotlib.pyplot')
    sys.path.insert(0, REF)
    from util import metric as ref_metric
    from util import util as ref_util
    from dataset import label_constants as lc
    # class counts evaluate() derives from the dataset name (util/metric.py:47-60)
    np.savez_compressed(os.path.join(OUT, 'metric_class_counts.npz'), names=np.array(['scannet_3d', 'matterport_3d_40', 'matterport_3d_80',
                        'matterport_3d_160', 'matterport_3d', 'nuscenes_3d']),
                        counts=np.array([len(lc.SCANNET_LABELS_20), len(lc.MATTERPORT_LABELS_40), len(lc.MATTERPORT_LABELS_80),
                                         len(lc.MATTERPORT_LABELS_160), len(lc.MATTERPORT_LABELS_21), len(lc.NUSCENES_LABELS_16)]))
    orig_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        for name, (C, ds, seed, nofeat) in {'scannet20': (20, 'scannet_3d', 31, False), 'mp160_nofeat': (160, 'matterport_3d_160', 32, True),
                                            'nuscenes16': (16, 'nuscenes_3d', 33, False)}.items():
            rng = np.random.RandomState(seed)
            n = 50000
            gt = rng.randint(0, C, n)
            gt[rng.rand(n) < 0.1] = 255
            gt[gt == 3] = 5                                      # a class that never occurs in gt
            pred = np.where(rng.rand(n) < 0.6, np.minimum(gt, C - 1), rng.randint(0, C, n))
            if nofeat:
                pred[rng.rand(n) < 0.05] = 256
            conf = ref_metric.confusion_matrix(pred.copy(), gt.copy(), C)
            miou = ref_metric.evaluate(pred.copy(), gt.copy(), stdout=False, dataset=ds)
            out = dict(pred=pred.astype(np.int32), gt=gt.astype(np.int32), C=C, confusion=conf.astype(np.int64), miou=np.float64(miou))
            if not nofeat:
                i_np, u_np, t_np = ref_util.intersectionAndUnion(pred.copy(), gt.copy(), C, 255)
                i_t, u_t, t_t = ref_util.intersectionAndUnionGPU(torch.from_numpy(pred.copy()), torch.from_numpy(gt.copy()), C, 255)
                assert np.array_equal(i_np, i_t.numpy()) and np.array_equal(u_np, u_t.numpy()) and np.array_equal(t_np, t_t.numpy())
                out.update(inter=i_np.astype(np.int64), union=u_np.astype(np.int64), target=t_np.astype(np.int64))
            np.savez_compressed(os.path.join(OUT, f'metric_{name}.npz'), **out)
            print('metric', name, 'mIoU', miou)
    finally:
        torch.Tensor.cuda = orig_cuda


def golden_loader():
    import functools
    import shutil
    import tempfile
    collections.Sequence = collections.abc.Sequence
    collections.Iterable = collections.abc.Iterable
    _stub_modules('SharedArray')
    sys.path.insert(0, REF)
    from dataset.feature_loader import FusedFeatureLoader
    orig_load = torch.load
    torch.load = functools.partial(orig_load, weights_only=False)
    tmp = tempfile.mkdtemp(prefix='osb_golden_')
    try:
        cases = {'train': dict(split='train', seed=51, legacy=False), 'val': dict(split='val', seed=52, legacy=False),
                 'train_legacy': dict(split='train', seed=53, legacy=True)}
        for name, c in cases.items():
            rng = np.random.RandomState(c['seed'])
            n, C = 3000, 16
            locs = (rng.rand(n, 3) * np.array([1.2, 1.0, 0.8])).astype(np.float32)
            colors = (rng.rand(n, 3) * 2 - 1).astype(np.float32)
            labels = rng.randint(0, 20, n).astype(np.float64)
            labels[rng.rand(n) < 0.1] = -100
            root = os.path.join(tmp, name, 'scannet_3d')
            os.makedirs(os.path.join(root, c['split']))
            featdir = os.path.join(tmp, name, 'feat')
            os.makedirs(featdir)
            torch.save((locs, colors, labels), os.path.join(root, c['split'], 'scene0000_00_vh_clean_2.pth'))
            mask_full = torch.from_numpy(rng.rand(n) < 0.4)
            M = int(mask_full.sum())
            feat = torch.from_numpy(rng.randn(M, C).astype(np.float16))
            blob = {'feat': feat, 'mask_full': mask_full}
            legacy_mask = None
            if c['legacy']:
                legacy_mask = torch.from_numpy(rng.rand(M) < 0.7)
                blob = {'feat': feat, 'mask': legacy_mask.nonzero()[:, 0], 'mask_full': mask_full}
            torch.save(blob, os.path.join(featdir, 'scene0000_00_0.pt'))
            loader = FusedFeatureLoader(datapath_prefix=root, datapath_prefix_feat=featdir, voxel_size=0.05, split=c['split'],
                                        aug=False, memcache_init=False, eval_all=(c['split'] != 'train'), input_color=False)
            np.random.seed(c['seed'] + 100)
            M_v, M_r = loader.voxelizer.get_transformation_matrix()
            np.random.seed(c['seed'] + 100)                       # same draws inside __getitem__ -> voxelize()
            item = loader[0]
            coords, feats, lab, feat_3d, mask = item[:5]
            out = dict(locs=locs, labels_in=labels, mask_full=mask_full.numpy(), feat=feat.numpy(), matrix=M_r @ M_v,
                       coords=coords.numpy(), feats=feats.numpy(), labels=lab.numpy(), feat_3d=feat_3d.numpy(), mask=mask.numpy(),
                       split=c['split'])
            if legacy_mask is not None:
                out['legacy_mask'] = legacy_mask.numpy()
            if len(item) > 5:
                out['inds_reverse'] = item[5].numpy()
            np.savez_compressed(os.path.join(OUT, f'loader_{name}.npz'), **out)
            print('loader', name, 'voxels', coords.shape[0], 'feat rows', feat_3d.shape[0], 'mask true', int(mask.sum()))
    finally:
        torch.load = orig_load
        shutil.rmtree(tmp, ignore_errors=True)


def _seed_where(pred, start=0):
    """first seed >= start whose Python `random` stream satisfies pred(random.Random(seed))"""
    import random
    s = start
    while not pred(random.Random(s)):
        s += 1
    return s


def _after_draws():
    import random
    return np.array([random.random() for _ in range(3)]), np.random.rand(3)


def golden_augment():
    """augment_{elastic,colour,point,fused}.npz: case k is stored under keys 'c<k>_*'."""
    import functools
    import random
    import shutil
    import tempfile
    collections.Sequence = collections.abc.Sequence
    collections.Iterable = collections.abc.Iterable
    _stub_modules('SharedArray')
    sys.path.insert(0, REF)
    import dataset.augmentation as t
    from dataset.feature_loader import FusedFeatureLoader
    from dataset.point_loader import Point3DLoader
    from openscene_b200 import synth

    def run(store, k, seed, fn, **inputs):
        random.seed(seed)
        np.random.seed(seed)
        out = fn(**{a: (b.copy() if isinstance(b, np.ndarray) else b) for a, b in inputs.items()})
        nxt_py, nxt_np = _after_draws()
        store[f'c{k}_seed'] = np.int64(seed)
        for a, b in inputs.items():
            store[f'c{k}_in_{a}'] = np.asarray(b)
        for a, b in out.items():
            store[f'c{k}_out_{a}'] = np.asarray(b)
        store[f'c{k}_next_py'], store[f'c{k}_next_np'] = nxt_py, nxt_np

    fires = lambda r: r.random() < 0.95            # noqa: E731
    skips = lambda r: r.random() >= 0.95           # noqa: E731

    # ---- elastic: float32 / float64 rooms, 1 and 2 points, the gate both ways, points on grid nodes and edges
    el = {}
    ed = t.ElasticDistortion(((0.2, 0.4), (0.8, 1.6)))
    room = synth.room_points((2.0, 1.6, 1.0), 3, 0.04, seed=5)
    room = room[::max(1, len(room) // 3000)]
    clouds = [room.astype(np.float32), room, np.array([[0.3, -1.2, 2.5]]), np.array([[0.0, 0.0, 0.0], [0.4, 0.6, 0.2]],
              dtype=np.float32), np.array([[0.0, 0.0, 0.0], [1.0, 0.6, 0.4], [0.2, 0.4, 0.6], [0.6, 0.2, 0.8]])]
    k = 0
    for ci, cl in enumerate(clouds):
        seed = _seed_where(fires, 100 * ci)
        run(el, k, seed, lambda pointcloud: {'coords': ed(pointcloud)}, pointcloud=cl)
        k += 1
    run(el, k, _seed_where(skips), lambda pointcloud: {'coords': ed(pointcloud)}, pointcloud=clouds[0])
    k += 1
    run(el, k, 7, lambda pointcloud: {'coords': t.ElasticDistortion(None)(pointcloud)}, pointcloud=clouds[1])
    np.savez_compressed(os.path.join(OUT, 'augment_elastic.npz'), n=np.int64(k + 1), **el)
    print('augment elastic cases', k + 1)

    # ---- colour / flip transforms one at a time: float32 and float64, both gate outcomes, clip edges, every hue sextant
    rng = np.random.RandomState(61)
    edge = np.array([[0, 0, 0], [255, 255, 255], [255, 0, 0], [255, 255, 0], [0, 255, 0], [0, 255, 255], [0, 0, 255],
                     [255, 0, 255], [128, 128, 128], [254.9, 0.1, 3.0], [255, 0, 1], [1, 0, 255], [7.5, 7.5, 7.5],
                     [200, 10, 10], [10, 200, 10], [10, 10, 200]], dtype=np.float64)
    cols64 = np.concatenate([edge, rng.rand(400, 3) * 255])
    coords = np.floor(rng.rand(len(cols64), 3) * [40, 30, 12])
    const = np.full((50, 3), 127.5)
    tf = {'flip': (t.RandomHorizontalFlip('z', False), 0.95), 'autocontrast': (t.ChromaticAutoContrast(), 0.2),
          'translation': (t.ChromaticTranslation(0.1), 0.95), 'jitter': (t.ChromaticJitter(0.05), 0.95),
          'hue_sat': (t.HueSaturationTranslation(0.5, 0.2), None)}
    co, k = {}, 0
    kinds = []
    for name, (tr, p) in tf.items():
        outcomes = [True] if p is None else [True, False]
        for dt in (np.float32, np.float64):
            for on in outcomes:
                for extra in range(2 if name in ('flip', 'hue_sat') else 1):
                    gate = (lambda r, p=p: r.random() < p) if on else (lambda r, p=p: r.random() >= p)
                    seed = _seed_where(gate if p is not None else (lambda r: True), 1000 * k + 17 * extra)
                    fn = lambda coords, feats, labels, tr=tr: dict(zip(('coords', 'feats', 'labels'), tr(coords, feats, labels)))
                    run(co, k, seed, fn, coords=coords.astype(dt), feats=cols64.astype(dt), labels=np.arange(len(cols64)) % 20)
                    kinds.append(name)
                    k += 1
    for dt in (np.float32, np.float64):                    # the constant-colour scene through the whole chain
        chain = t.Compose([t.RandomHorizontalFlip('z', False), t.ChromaticAutoContrast(), t.ChromaticTranslation(0.1),
                           t.ChromaticJitter(0.05), t.HueSaturationTranslation(0.5, 0.2)])
        seed = _seed_where(lambda r: r.random() < 0.95 and [r.random() for _ in range(2)] and r.random() < 0.2)
        fn = lambda coords, feats, labels, chain=chain: dict(zip(('coords', 'feats', 'labels'), chain(coords, feats, labels)))
        with np.errstate(invalid='ignore', divide='ignore'):
            run(co, k, seed, fn, coords=coords[:50].astype(dt), feats=const.astype(dt), labels=np.arange(50) % 20)
        kinds.append('chain')
        k += 1
    np.savez_compressed(os.path.join(OUT, 'augment_colour.npz'), n=np.int64(k), kinds=np.array(kinds), **co)
    print('augment colour cases', k)

    # ---- loader items through the reference's own loaders
    orig_load = torch.load
    torch.load = functools.partial(orig_load, weights_only=False)
    tmp = tempfile.mkdtemp(prefix='osb_golden_aug_')
    try:
        pt, fu = {}, {}
        cases = [dict(n=3000, dt=np.float32, color=False, seed=71), dict(n=3000, dt=np.float64, color=True, seed=72),
                 dict(n=2500, dt=np.float32, color=True, seed=73, const=True), dict(n=1, dt=np.float32, color=True, seed=74),
                 dict(n=2, dt=np.float64, color=True, seed=75)]
        for k, c in enumerate(cases):
            rng = np.random.RandomState(c['seed'])
            n = c['n']
            locs = (rng.rand(n, 3) * np.array([2.4, 2.0, 1.2])).astype(c['dt'])
            colors = (rng.rand(n, 3) * 2 - 1).astype(c['dt'])
            if c.get('const'):
                colors[:] = 0
            else:
                colors[:3] = np.array([[-1, -1, -1], [1, 1, 1], [1, -1, 0]], dtype=c['dt'])[:min(3, n)]
            labels = rng.randint(0, 20, n).astype(np.float64)
            labels[rng.rand(n) < 0.1] = -100
            root = os.path.join(tmp, f'p{k}', 'scannet_3d')
            os.makedirs(os.path.join(root, 'train'))
            featdir = os.path.join(tmp, f'p{k}', 'feat')
            os.makedirs(featdir)
            torch.save((locs, colors, labels), os.path.join(root, 'train', 'scene0000_00_vh_clean_2.pth'))
            mask_full = torch.from_numpy(rng.rand(n) < 0.5)
            mask_full[0] = True
            feat = torch.from_numpy(rng.randn(int(mask_full.sum()), 16).astype(np.float16))
            torch.save({'feat': feat, 'mask_full': mask_full}, os.path.join(featdir, 'scene0000_00_0.pt'))
            lab_in = labels.copy()
            lab_in[lab_in == -100] = 255
            lab_in = lab_in.astype(np.uint8)
            pl = Point3DLoader(datapath_prefix=root, voxel_size=0.05, split='train', aug=True, input_color=c['color'])
            fl = FusedFeatureLoader(datapath_prefix=root, datapath_prefix_feat=featdir, voxel_size=0.05, split='train',
                                    aug=True, input_color=c['color'])
            ins = dict(locs=locs, feats=(colors + 1.) * 127.5, labels=lab_in, colors=colors, input_color=c['color'])
            fns = {'point': lambda **_: dict(zip(('coords', 'feats', 'labels'), pl[0])),
                   'fused': lambda **_: dict(zip(('coords', 'feats', 'labels', 'feat_3d', 'mask'), fl[0]))}
            for store, kind in ((pt, 'point'), (fu, 'fused')):
                seed = _seed_where(fires, 10 * c['seed'] + (kind == 'fused'))
                run(store, k, seed, fns[kind], **ins)
                if kind == 'fused':
                    store[f'c{k}_in_feat'], store[f'c{k}_in_mask_full'] = feat.numpy(), mask_full.numpy()
            print('augment items', k, 'points', n, 'voxels', pt[f'c{k}_out_coords'].shape[0])
        np.savez_compressed(os.path.join(OUT, 'augment_point.npz'), n=np.int64(len(cases)), **pt)
        np.savez_compressed(os.path.join(OUT, 'augment_fused.npz'), n=np.int64(len(cases)), **fu)
    finally:
        torch.load = orig_load
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    todo = sys.argv[1:] or ['voxelizer', 'unet', 'fusion', 'metric', 'loader', 'augment']
    for nm in todo:
        {'voxelizer': golden_voxelizer, 'unet': golden_unet, 'fusion': golden_fusion, 'metric': golden_metric, 'loader': golden_loader,
         'augment': golden_augment}[nm]()
