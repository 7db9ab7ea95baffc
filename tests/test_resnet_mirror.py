"""The table-driven ResNet mirror (openscene_b200/resnet.py) against the reference's ``models/resnet_base.py`` as recorded in
tests/golden/live_resnets.npz (scripts/make_golden_resnet.py): the same state-dict keys, shapes and seed-0 weights, so
checkpoints load with ``strict=True`` either way.  Where a reference checkout is named by OSB_REFERENCE_ROOT, its own
ResNet14 / ResNet50 are built on this package and their forward runs to the end (on the CPU oracle: this package has no
CPU path).  The GPU forward and training step are in tests/test_gpu_pool_modules.py."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests.test_reference_models_on_product import weight_fingerprint
from tests.util import digest, golden

ARCHS = ['ResNet14', 'ResNet18', 'ResNet34', 'ResNet50', 'ResNet101']
LOGIT_ARCHS = ['ResNet14', 'ResNet18']
OUT_CHANNELS = 13


def resnet_cloud():
    """two scenes spanning tensor stride 192 (so conv5 and the global pooling see several rows per scene)"""
    coords = synth.random_cloud(6000, 400, seed=21, batch=2)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(22))
    return coords, feats


def oracle_me():
    """the CPU oracle as an ``ME`` namespace whose MinkowskiLinear also takes the dense ``[B, C]`` the global pooling returns
    (the oracle's own MinkowskiLinear reads ``x.F``); the head's parameters and arithmetic are the oracle's"""
    from oracle import me_cpu

    class MinkowskiLinear(me_cpu.MinkowskiLinear):
        def forward(self, x):
            return self.linear(x) if torch.is_tensor(x) else super().forward(x)

    ns = me_cpu.as_module()
    ns.MinkowskiLinear = MinkowskiLinear
    return ns


def mirror(arch, ME=None):
    from openscene_b200 import resnet
    torch.manual_seed(0)
    return resnet.resnet(arch, 3, OUT_CHANNELS, ME=ME)


@pytest.mark.parametrize('arch', ARCHS)
def test_mirror_matches_the_reference_state_dict(arch):
    g = golden('live_resnets.npz')
    sd = mirror(arch).state_dict()
    keys, shapes, weights = [d.decode() for d in g['archs'][ARCHS.index(arch)]]
    assert digest(list(sd.keys())) == keys
    assert digest([str(tuple(v.shape)) for v in sd.values()]) == shapes
    assert digest([weight_fingerprint(v) for v in sd.values()]) == weights
    mirror(arch).load_state_dict(sd, strict=True)


def test_mirror_forward_on_the_oracle_matches_the_golden_logits():
    """the mirror's topology and dataflow on the fp64 oracle reproduce the reference forward's logits"""
    from oracle import me_cpu
    g = golden('live_resnets.npz')
    coords, feats = resnet_cloud()
    for arch, ref in zip(LOGIT_ARCHS, g['logits']):
        model = mirror(arch)
        m64 = mirror(arch, ME=oracle_me()).double().eval()
        m64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in model.state_dict().items()})
        with torch.no_grad():
            y = m64(me_cpu.SparseTensor(feats.double(), torch.from_numpy(coords))).numpy()
        assert np.allclose(y, ref, rtol=1e-12, atol=1e-12), arch


def _reference_resnet_base():
    ref = os.environ.get('OSB_REFERENCE_ROOT')
    if not ref or not os.path.exists(os.path.join(ref, 'models', 'resnet_base.py')):
        pytest.skip('no reference checkout (OSB_REFERENCE_ROOT)')
    sys.modules.pop('resnet_base', None)
    sys.path.insert(0, os.path.join(ref, 'models'))
    try:
        return importlib.import_module('resnet_base')
    finally:
        sys.path.pop(0)
        sys.modules.pop('resnet_base', None)


@pytest.mark.parametrize('arch', ['ResNet14', 'ResNet50'])
def test_reference_resnet_builds_on_the_package_and_runs_to_the_end(arch):
    import MinkowskiEngine                                                  # noqa: F401  this repository's package
    from oracle import me_cpu
    rb = _reference_resnet_base()
    torch.manual_seed(0)
    model = getattr(rb, arch)(3, OUT_CHANNELS)
    sd = model.state_dict()
    assert list(sd.keys()) == list(mirror(arch).state_dict().keys())
    assert all(torch.equal(a, b) for a, b in zip(sd.values(), mirror(arch).state_dict().values()))
    # the reference's own forward (ResNetBase.forward) end to end: global pooling -> MinkowskiLinear on a dense tensor
    m64 = mirror(arch, ME=oracle_me()).double().eval()
    m64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in sd.items()})
    coords, feats = resnet_cloud()
    with torch.no_grad():
        y = rb.ResNetBase.forward(m64, me_cpu.SparseTensor(feats.double(), torch.from_numpy(coords)))
    assert y.shape == (2, OUT_CHANNELS) and torch.isfinite(y).all()
