"""Record the reference's sparse ResNets (models/resnet_base.py) as tests/golden/live_resnets.npz:
  - for every class (ResNet14/18/34/50/101) built with torch.manual_seed(0) on THIS repository's MinkowskiEngine package:
    digests of its state-dict keys, shapes and seeded weight fingerprints (as make_golden_live.py records MinkUNet);
  - for ResNet14 and ResNet18: the fp64 logits of the reference's own forward on the CPU oracle (oracle/me_cpu.py, its
    MinkowskiLinear taking the dense output of the global pooling: tests/test_resnet_mirror.oracle_me), with
    those seed-0 weights, on a seeded two-scene cloud (tests/test_resnet_mirror.py builds the same cloud).
Usage: OSB_REFERENCE_ROOT=<reference checkout> python scripts/make_golden_resnet.py"""
import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ['OSB_REFERENCE_ROOT']
OUT = os.path.join(ROOT, 'tests', 'golden', 'live_resnets.npz')

from tests.test_reference_models_on_product import weight_fingerprint   # noqa: E402
from tests.test_resnet_mirror import ARCHS, LOGIT_ARCHS, OUT_CHANNELS, oracle_me, resnet_cloud   # noqa: E402
from tests.util import digest                                            # noqa: E402


def _reference_module(me_pkg):
    """models/resnet_base.py imported with ``MinkowskiEngine`` resolving to me_pkg (a fresh import each time)"""
    for k in [k for k in sys.modules if k == 'MinkowskiEngine' or k.startswith('MinkowskiEngine.') or k == 'resnet_base']:
        del sys.modules[k]
    if me_pkg == 'oracle':
        from oracle import me_cpu
        me = me_cpu.install_as_minkowski_engine()
        shim = types.ModuleType('MinkowskiEngine')                   # the oracle with the dense-input linear head
        shim.__dict__.update({k: v for k, v in me.__dict__.items() if not k.startswith('__')})
        shim.MinkowskiLinear = oracle_me().MinkowskiLinear
        sys.modules['MinkowskiEngine'] = shim
    sys.path.insert(0, os.path.join(REF, 'models'))
    try:
        return importlib.import_module('resnet_base')
    finally:
        sys.path.pop(0)


def main():
    sys.path.insert(0, ROOT)
    rb = _reference_module('product')
    archs, states = [], {}
    for arch in ARCHS:
        torch.manual_seed(0)
        sd = getattr(rb, arch)(3, OUT_CHANNELS).state_dict()
        archs.append([digest(list(sd.keys())), digest([str(tuple(v.shape)) for v in sd.values()]),
                      digest([weight_fingerprint(v) for v in sd.values()])])
        states[arch] = {k: v.clone() for k, v in sd.items()}
    rbo = _reference_module('oracle')
    from oracle import me_cpu
    coords, feats = resnet_cloud()
    logits = []
    for arch in LOGIT_ARCHS:
        model = getattr(rbo, arch)(3, OUT_CHANNELS).double().eval()
        model.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in states[arch].items()}, strict=True)
        with torch.no_grad():
            y = model(me_cpu.SparseTensor(feats.double(), torch.from_numpy(coords)))
        assert y.shape == (2, OUT_CHANNELS) and torch.isfinite(y).all()
        logits.append(y.numpy())
    np.savez_compressed(OUT, archs=np.array(archs, dtype='S64'), logits=np.stack(logits))
    print('wrote', OUT)


if __name__ == '__main__':
    main()
