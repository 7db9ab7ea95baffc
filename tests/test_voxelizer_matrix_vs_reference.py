"""Host half of the drop-in voxeliser against what the REFERENCE's own class returned (tests/golden/live_voxelizer.npz,
recorded by scripts/make_golden_live.py on the cases below).

``openscene_b200.voxelize.Voxelizer.get_transformation_matrix`` must consume the global NumPy RNG exactly as
``dataset/voxelizer.py:46-76`` does -- the loaders seed / share that stream (dataset/point_loader.py:58-61), so a different draw
order would change every augmentation after it.  Compared bit for bit, matrices and RNG state, over the constructor forms the
reference's loaders use; the NumPy oracle (oracle/voxelize_ref.py) is held to the same reference on random clouds beyond the four
original fixtures."""
import numpy as np
import pytest

from tests.util import digest, golden

ROT = ((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi))        # point_loader.py:58-61
FORMS = [
    dict(voxel_size=0.02, use_augmentation=True, scale_augmentation_bound=(0.9, 1.1), rotation_augmentation_bound=ROT),
    dict(voxel_size=0.05, use_augmentation=True, scale_augmentation_bound=(0.9, 1.1), rotation_augmentation_bound=ROT),
    dict(voxel_size=0.02, use_augmentation=False, scale_augmentation_bound=(0.9, 1.1), rotation_augmentation_bound=ROT),
    dict(voxel_size=0.02, use_augmentation=True, scale_augmentation_bound=None, rotation_augmentation_bound=ROT),
    dict(voxel_size=0.02, use_augmentation=True, scale_augmentation_bound=(0.9, 1.1), rotation_augmentation_bound=None),
    dict(voxel_size=0.02, use_augmentation=True, scale_augmentation_bound=(0.9, 1.1),
         rotation_augmentation_bound=(None, (-0.1, 0.1), (-np.pi, np.pi))),
]
TRANS = ((-0.2, 0.2), (-0.2, 0.2), (0, 0))


def voxel_clouds():
    """[(trial, points, voxel size, augmentation on)]: dense clouds with duplicates, negative coordinates, fp32 and fp64."""
    rng = np.random.RandomState(2024)
    out = []
    for trial in range(12):
        n = int(rng.randint(500, 6000))
        extent, shift = float(rng.uniform(0.3, 5.0)), float(rng.uniform(-3.0, 1.0))
        dtype = np.float32 if trial % 3 == 0 else np.float64
        pts = (rng.rand(n, 3) * extent + shift).astype(dtype)
        out.append((trial, pts, float(rng.choice([0.02, 0.05, 0.1])), trial % 2 == 0))
    return out


@pytest.mark.parametrize('form', range(len(FORMS)))
def test_matrix_and_rng_stream_equal_the_reference(form):
    from openscene_b200.voxelize import Voxelizer as Mine
    g = golden('live_voxelizer.npz')
    mine = Mine(**dict(FORMS[form], clip_bound=None, translation_augmentation_ratio_bound=TRANS, ignore_label=255))
    mats = []
    for seed in range(25):
        np.random.seed(seed)
        b_v, b_r = mine.get_transformation_matrix()
        tail_mine = np.random.rand(4)                    # what the next consumer of the stream would see: the same RNG use
        mats.append(np.stack([b_v, b_r, np.r_[tail_mine, np.zeros(12)].reshape(4, 4)]))
    assert digest(np.stack(mats)) == g['forms'][form].decode(), form


def test_oracle_equals_the_reference_on_random_clouds():
    """oracle/voxelize_ref.py vs the reference's voxelize() beyond the original fixtures: dense clouds with many duplicates,
    negative coordinates, fp32 and fp64 inputs, augmentation on and off."""
    from oracle import voxelize_ref
    g = golden('live_voxelizer.npz')
    for trial, pts, vsize, aug in voxel_clouds():
        got = voxelize_ref.voxelize(pts, g['rigid'][trial])[:3]          # coordinates, inds, inverse
        assert [digest(a) for a in got] == [d.decode() for d in g['clouds'][trial]], trial
