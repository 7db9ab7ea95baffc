"""Record what the reference's own functions return on the cases the three tests below define, as tests/golden/live_*.npz
(SHA-256 digests of exact results, tests/util.digest): fusion_util.py's compute_mapping, util/metric.py and
util/util.py's metrics, dataset/voxelizer.py's matrices, RNG use and voxelize(), and models/mink_unet.py / disnet.py state
dicts and the names the factory refuses.  The tests hold the oracles and the product to these, without the reference tree.
Usage: OSB_REFERENCE_ROOT=<reference checkout> python scripts/make_golden_live.py"""
import collections
import collections.abc
import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ['OSB_REFERENCE_ROOT']
OUT = os.path.join(ROOT, 'tests', 'golden')

from tests.test_oracles_vs_reference_live import fusion_cases, metric_cases                    # noqa: E402
from tests.test_reference_models_on_product import ALL_ARCHS, weight_fingerprint                # noqa: E402
from tests.test_voxelizer_matrix_vs_reference import FORMS, ROT, TRANS, voxel_clouds            # noqa: E402
from tests.util import digest                                                                    # noqa: E402


def _stub(*names):
    for nm in names:
        parts = nm.split('.')
        for i in range(1, len(parts) + 1):
            sub = '.'.join(parts[:i])
            if sub not in sys.modules:
                sys.modules[sub] = types.ModuleType(sub)
            if i > 1:
                setattr(sys.modules['.'.join(parts[:i - 1])], parts[i - 1], sys.modules[sub])


def fusion():
    _stub('tensorflow', 'tensorflow.io', 'tensorflow.compat', 'tensorflow.compat.v1')   # imported, never used by the mapper
    sys.path.insert(0, os.path.join(REF, 'scripts', 'feature_fusion'))
    import fusion_util
    maps, vis = [], []                                   # every view of every case, in order
    for seed, pts, poses, depths, intr, cut, thres in fusion_cases():
        mapper = fusion_util.PointCloudToImageMapper(image_dim=(320, 240), intrinsics=intr, visibility_threshold=thres, cut_bound=cut)
        for pose, depth in zip(poses, depths):
            m = mapper.compute_mapping(pose, pts, depth)
            maps.append(digest(m))
            vis.append(int(m[:, 2].sum()))
    np.savez_compressed(os.path.join(OUT, 'live_fusion_mapping.npz'), maps=np.array(maps, dtype='S64'), vis=np.array(vis))


def metric():
    _stub('open3d', 'clip', 'matplotlib', 'matplotlib.patches', 'matplotlib.pyplot')
    sys.path.insert(0, REF)
    torch.Tensor.cuda = lambda self, *a, **k: self           # intersectionAndUnionGPU calls .cuda()
    from util import metric as m, util as u
    conf, miou, iut = [], [], []                         # per case; iut: intersection, union, target ('' without them)
    for seed, C, ds, pred, gt, nofeat in metric_cases():
        conf.append(digest(m.confusion_matrix(pred.copy(), gt.copy(), C)))
        miou.append(float(m.evaluate(pred.copy(), gt.copy(), stdout=False, dataset=ds)))
        iut.append(['', '', ''])
        if not nofeat:
            i_np, u_np, t_np = u.intersectionAndUnion(pred.copy(), gt.copy(), C, 255)
            i_t, u_t, t_t = u.intersectionAndUnionGPU(torch.from_numpy(pred.copy()), torch.from_numpy(gt.copy()), C, 255)
            for k, (a, b) in enumerate(((i_np, i_t), (u_np, u_t), (t_np, t_t))):
                assert np.array_equal(a.astype(np.int64), b.numpy().astype(np.int64))
                iut[-1][k] = digest(a)
    np.savez_compressed(os.path.join(OUT, 'live_metric.npz'), conf=np.array(conf, dtype='S64'), miou=np.array(miou),
                        iut=np.array(iut, dtype='S64'))


def voxelizer():
    collections.Sequence = collections.abc.Sequence      # dataset/voxelization_utils.py:6 (Python 3.12)
    collections.Iterable = collections.abc.Iterable      # dataset/voxelizer.py:55
    sys.path.insert(0, REF)
    from dataset.voxelizer import Voxelizer
    out = {}
    forms = []                                           # per form: digest of [seed][rigid matrix, rotation, next 4 draws]
    for form in FORMS:
        ref = Voxelizer(**dict(form, clip_bound=None, translation_augmentation_ratio_bound=TRANS, ignore_label=255))
        mats = []
        for seed in range(25):
            np.random.seed(seed)
            a_v, a_r = ref.get_transformation_matrix()
            mats.append(np.stack([a_v, a_r, np.r_[np.random.rand(4), np.zeros(12)].reshape(4, 4)]))
        forms.append(digest(np.stack(mats)))
    out['forms'] = np.array(forms, dtype='S64')
    rigid, clouds = [], []                                        # [trial]: matrix, (coordinates, inds, inverse) digests
    for trial, pts, vsize, aug in voxel_clouds():
        n = len(pts)
        vox = Voxelizer(voxel_size=vsize, clip_bound=None, use_augmentation=aug, scale_augmentation_bound=(0.9, 1.1),
                        rotation_augmentation_bound=ROT, translation_augmentation_ratio_bound=TRANS)
        np.random.seed(trial)
        M_v, M_r = vox.get_transformation_matrix()
        np.random.seed(trial)
        coords_aug, _, _, inds_rec, inds = vox.voxelize(pts, np.zeros((n, 3), np.float32), np.zeros(n, np.int64), return_ind=True)
        rigid.append((M_r @ M_v) if aug else M_v)
        clouds.append([digest(coords_aug), digest(inds), digest(inds_rec)])
    out['rigid'], out['clouds'] = np.array(rigid), np.array(clouds, dtype='S64')
    np.savez_compressed(os.path.join(OUT, 'live_voxelizer.npz'), **out)


def models():
    sys.path.insert(0, ROOT)
    import MinkowskiEngine  # noqa: F401  (this repository's package: the reference's model files import it)
    sys.path.insert(0, REF)
    mu = importlib.import_module('models.mink_unet')
    dn = importlib.import_module('models.disnet')
    out, archs = {}, []                                  # archs: [ALL_ARCHS]: digests of keys, shapes, weight fingerprints
    for arch in ALL_ARCHS:
        torch.manual_seed(0)
        sd = mu.mink_unet(in_channels=3, out_channels=20, D=3, arch=arch).state_dict()
        archs.append([digest(list(sd.keys())), digest([str(tuple(v.shape)) for v in sd.values()]),
                      digest([weight_fingerprint(v) for v in sd.values()])])
    out['archs'] = np.array(archs, dtype='S64')
    rejected = []                                        # names the reference's factory refuses to build
    for arch in ('MinkUNet50', 'MinkUNet101', 'nonsense'):
        try:
            mu.mink_unet(arch=arch)
        except Exception:       # noqa: BLE001
            rejected.append(arch)
    out['rejected'] = np.array(rejected, dtype='S16')
    disnet = []                                          # openseg, lseg: digest of the state-dict keys
    for ext, c in (('openseg', 768), ('lseg', 512)):
        net = dn.DisNet(cfg=types.SimpleNamespace(arch_3d='MinkUNet18A', feature_2d_extractor=ext))
        disnet.append(digest(list(net.state_dict().keys())))
        assert net.net3d.final.kernel.shape == (96, c)
    out['disnet'] = np.array(disnet, dtype='S64')
    np.savez_compressed(os.path.join(OUT, 'live_models.npz'), **out)


if __name__ == '__main__':
    fusion()
    metric()
    voxelizer()
    models()
    print('wrote', OUT)
