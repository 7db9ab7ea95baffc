"""The CPU oracles against what the REFERENCE's own functions returned on random cases beyond the original fixtures
(tests/golden/live_*.npz, recorded by scripts/make_golden_live.py on the cases below).

* oracle/fusion_ref.compute_mapping  vs  scripts/feature_fusion/fusion_util.py: PointCloudToImageMapper.compute_mapping
* oracle/metric_ref                  vs  util/metric.py (confusion_matrix, evaluate) and util/util.py (intersectionAndUnion[GPU])
Bit-exact (integer work); mIoU to 1e-12."""
import numpy as np
import pytest

from tests.util import digest, golden


def fusion_cases():
    """[(seed, pts, poses, depths, intrinsics, cut_bound, visibility_threshold)] for seeds 100-107."""
    from openscene_b200.synth import fusion_case
    out = []
    for seed in range(100, 108):
        with_depth = seed % 3 != 0
        pts, poses, depths, intr = fusion_case(seed, 2500 + 300 * (seed % 5), with_depth)
        out.append((seed, pts, poses, depths, intr, [0, 5, 10, 20][seed % 4], [0.25, 0.1, 0.5][seed % 3]))
    return out


def metric_cases():
    """[(seed, n_classes, dataset name, pred, gt, has no-feature points)]: 15 % ignore labels, one class absent from gt."""
    out = []
    for seed, (C, ds) in enumerate([(20, 'scannet_3d'), (21, 'matterport_3d'), (40, 'matterport_3d_40'), (80, 'matterport_3d_80'),
                                    (160, 'matterport_3d_160'), (16, 'nuscenes_3d')]):
        rng = np.random.RandomState(500 + seed)
        n = 20000
        gt = rng.randint(0, C, n)
        gt[rng.rand(n) < 0.15] = 255
        gt[gt == (seed % C)] = (seed + 1) % C
        pred = np.where(rng.rand(n) < 0.5, np.minimum(gt, C - 1), rng.randint(0, C, n))
        nofeat = seed % 2 == 1
        if nofeat:
            pred[rng.rand(n) < 0.07] = 256
        out.append((seed, C, ds, pred, gt, nofeat))
    return out


def test_fusion_mapping_oracle_equals_the_reference_on_random_views():
    from oracle import fusion_ref
    g = golden('live_fusion_mapping.npz')
    v = 0
    for seed, pts, poses, depths, intr, cut, thres in fusion_cases():
        for pose, depth in zip(poses, depths):
            got = fusion_ref.compute_mapping(pose, pts, depth, intr, (320, 240), cut, thres)
            assert digest(got) == g['maps'][v].decode(), seed
            v += 1
    assert v == len(g['maps']) and g['vis'].sum() > 5000                                       # the cases exercise the visible branch


def test_metric_oracles_equal_the_reference_on_random_labels():
    from oracle import metric_ref
    g = golden('live_metric.npz')
    for seed, C, ds, pred, gt, nofeat in metric_cases():
        assert digest(metric_ref.confusion_matrix(pred, gt, C)) == g['conf'][seed].decode(), ds
        assert metric_ref.mean_iou(pred, gt, C)[0] == pytest.approx(float(g['miou'][seed]), rel=1e-12), ds
        if not nofeat:
            for a, want in zip(metric_ref.intersection_and_union(pred, gt, C), g['iut'][seed]):
                assert digest(a) == want.decode(), ds
