"""Matching (run/evaluate.py:288-323) and the voxeliser (dataset/voxelizer.py) on the GPU against the oracle
and against the vectors produced by the reference's own voxeliser.  Scores are judged against their per-score fp64 bound
(tests/match_ref.py), labels by the label rule on the kernel's own scores."""
import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests import match_ref as M
from tests.util import golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _feats(n, c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, c, generator=g) * (0.2 + torch.rand(n, 1, generator=g))


@pytest.mark.parametrize('k,c', [(20, 768), (160, 768), (21, 512)])
def test_distill_and_fusion_scores(k, c):
    from openscene_b200 import matching
    from oracle import matching as om
    f = _feats(3000, c, 0)
    inv = torch.randint(0, 3000, (7000,), generator=torch.Generator().manual_seed(1))
    text = torch.from_numpy(synth.text_embeddings(k, c))
    s, l = matching.match_distill(f.to(DEV), inv.to(DEV), text.to(DEV))
    sr, lr = om.match_distill(f, inv, text)
    assert s.dtype == torch.float16 and s.shape == (7000, k) and l.dtype == torch.int64
    assert M.check_scores(s, f.to(DEV), inv.to(DEV), text.to(DEV), False, 'tc') <= 1.0
    M.check_labels(s, l)
    # the oracle's fp32 product lies within the same bound (it is the reference's arithmetic, not a neighbour of it)
    assert M.check_scores(sr, f, inv, text, False, 'tc') <= 1.0
    assert torch.equal(lr, M.label_rule(sr)[0])
    s2, l2 = matching.match_fusion(f.half().to(DEV), inv.to(DEV), text.to(DEV))
    assert M.check_scores(s2, f.half().to(DEV), inv.to(DEV), text.to(DEV), False, 'tc') <= 1.0
    M.check_labels(s2, l2)


def test_ensemble_path():
    from openscene_b200 import matching
    from oracle import matching as om
    f3, f2 = _feats(2500, 768, 2), _feats(2500, 768, 3).half()
    inv = torch.randint(0, 2500, (6000,), generator=torch.Generator().manual_seed(4))
    text = torch.from_numpy(synth.text_embeddings(160))
    s, l, fe, m = matching.match_ensemble(f3.to(DEV), f2.to(DEV), inv.to(DEV), text.to(DEV), return_features=True)
    sr, lr, fer, mr = om.match_ensemble(f3, f2, inv, text)
    # a choice may differ from fp64 only where the two maxima's bound intervals overlap; the feature is the chosen row
    M.check_ensemble(s, l, fe, m, f3.to(DEV), f2.to(DEV), inv.to(DEV), text.to(DEV), 'tc')
    M.check_ensemble(sr, lr, fer, mr, f3, f2, inv, text, 'tc')          # the oracle obeys the same rule


@pytest.mark.parametrize('case', ['aug_f64', 'noaug_f32', 'dups_f64', 'neg_f64'])
def test_voxelizer_matches_reference_vectors(case):
    from openscene_b200.voxelize import voxelize_points
    g = golden(f'voxelizer_{case}.npz')
    cv, inds, inv, _ = voxelize_points(torch.from_numpy(g['points']).to(DEV), g['matrix'])
    assert np.array_equal(cv.cpu().numpy().astype(np.float64), g['coords_vox'])
    assert np.array_equal(inds.cpu().numpy(), g['inds'])
    assert np.array_equal(inv.cpu().numpy(), g['inds_reverse'])


def test_voxelizer_class_interface_and_properties():
    from openscene_b200.voxelize import Voxelizer
    from oracle import voxelize_ref
    pts = synth.room_points((1.0, 0.8, 0.6), 2, seed=3)
    n = len(pts)
    vox = Voxelizer(voxel_size=0.02, use_augmentation=True, scale_augmentation_bound=(0.9, 1.1),
                    rotation_augmentation_bound=((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi)))
    np.random.seed(5)
    M_v, M_r = vox.get_transformation_matrix()
    np.random.seed(5)
    feats, labels = np.ones((n, 3), np.float32), np.arange(n)
    c, f, l, inv, inds = vox.voxelize(pts, feats, labels, return_ind=True)
    cr, ir, invr, _ = voxelize_ref.voxelize(pts, M_r @ M_v)
    assert np.array_equal(c, cr) and np.array_equal(inds, ir) and np.array_equal(inv, invr)
    # size-independent properties: unique rows, inverse reconstructs, first occurrence
    assert len(np.unique(c, axis=0)) == len(c)
    assert np.array_equal(c[inv][inds], c)
    assert (inds[inv] <= np.arange(n)).all()
    assert np.array_equal(l, inds)
