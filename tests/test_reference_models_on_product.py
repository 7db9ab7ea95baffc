"""The model files of the reference (``models/mink_unet.py`` / ``models/disnet.py``) imported on top of THIS repository's
``MinkowskiEngine`` package give the state-dict keys, shapes and seeded weights recorded in tests/golden/live_models.npz
(scripts/make_golden_live.py); the table-driven mirror ``openscene_b200/minkunet.py`` must give exactly the same, so
checkpoints written by one load with ``strict=True`` (run/evaluate.py:168) into the other."""
import types

import numpy as np
import pytest
import torch

from tests.util import digest, golden

ALL_ARCHS = ['MinkUNet14A', 'MinkUNet14B', 'MinkUNet14C', 'MinkUNet14D', 'MinkUNet18A', 'MinkUNet18B', 'MinkUNet18D',
             'MinkUNet34A', 'MinkUNet34B', 'MinkUNet34C']


def weight_fingerprint(t):
    """Order-sensitive float64 summary of a seeded tensor: equal weights give equal fingerprints."""
    v = t.detach().double().flatten()
    w = np.arange(1, v.numel() + 1, dtype=np.float64)
    return '%.17g %.17g' % (float(v.sum()), float((v.numpy() * w).sum()))


def _mirror(arch, out_channels):
    from openscene_b200 import minkunet
    torch.manual_seed(0)
    return minkunet.mink_unet(in_channels=3, out_channels=out_channels, D=3, arch=arch)


def _check_against_reference(arch):
    g = golden('live_models.npz')
    sd = _mirror(arch, 20).state_dict()
    keys, shapes, weights = [d.decode() for d in g['archs'][ALL_ARCHS.index(arch)]]
    assert digest(list(sd.keys())) == keys
    assert digest([str(tuple(v.shape)) for v in sd.values()]) == shapes
    assert digest([weight_fingerprint(v) for v in sd.values()]) == weights        # same seed, order, init rule


@pytest.mark.parametrize('arch', ['MinkUNet18A', 'MinkUNet34C'])
def test_reference_model_file_builds_on_the_product_package(arch):
    _check_against_reference(arch)
    g = golden(f'unet_{arch}.npz')
    model = _mirror(arch, 768)
    sd = model.state_dict()
    assert list(sd.keys()) == g['state_keys'].tolist()
    assert [str(tuple(v.shape)) for v in sd.values()] == g['state_shapes'].tolist()
    assert sum(p.numel() for p in model.parameters()) == int(g['n_params'])
    # a checkpoint loads strictly, with or without the DDP prefix (run/evaluate.py:177-191)
    _mirror(arch, 768).load_state_dict(sd, strict=True)


def test_reference_disnet_on_the_product_package():
    from openscene_b200 import minkunet
    g = golden('live_models.npz')
    for ext, c, keys in zip(('openseg', 'lseg'), (768, 512), g['disnet']):
        net = minkunet.DisNet(cfg=types.SimpleNamespace(arch_3d='MinkUNet18A', feature_2d_extractor=ext))
        assert digest(list(net.state_dict().keys())) == keys.decode()
        assert tuple(net.net3d.final.kernel.shape) == (96, c)       # the reference's head shapes (checked when recorded)


@pytest.mark.parametrize('arch', [a for a in ALL_ARCHS if a not in ('MinkUNet18A', 'MinkUNet34C')])
def test_every_factory_architecture_matches_the_mirror(arch):
    """The eight other names `mink_unet()` accepts (models/mink_unet.py:241-263): the reference's class on the product package and
    the table-driven mirror give the same state-dict keys, shapes and seeded weights."""
    _check_against_reference(arch)


def test_factory_rejects_what_the_reference_rejects():
    """`mink_unet(arch=...)` raises for names outside its list -- MinkUNet50 / MinkUNet101 included: the reference defines those
    classes (models/mink_unet.py:191-199) but gives them no PLANES, so they cannot be constructed there either."""
    from openscene_b200 import minkunet
    rejected = [a.decode() for a in golden('live_models.npz')['rejected']]       # recorded from the reference's factory
    assert rejected == ['MinkUNet50', 'MinkUNet101', 'nonsense']
    for arch in rejected:
        with pytest.raises(Exception):
            minkunet.mink_unet(arch=arch)
