"""Drop-in ``MinkowskiEngine`` for OpenScene, backed by libosb200 (H100 / sm_90a).

``import MinkowskiEngine as ME`` in the reference's models/mink_unet.py:25, models/resnet_base.py:27,
run/distill.py:18 and run/evaluate.py:18 resolves here when this repository is on PYTHONPATH.
"""
from openscene_b200.me import *  # noqa: F401,F403
from openscene_b200.me import (CoordinateMapKey, MinkowskiAvgPooling, MinkowskiBatchNorm, MinkowskiConvolution,
                               MinkowskiConvolutionTranspose, MinkowskiGlobalAvgPooling, MinkowskiGlobalMaxPooling,
                               MinkowskiGlobalSumPooling, MinkowskiLinear, MinkowskiMaxPooling, MinkowskiReLU,
                               MinkowskiSumPooling, SparseTensor, __version__, cat)
from openscene_b200.coords import CoordinateManager  # noqa: F401
from . import modules, utils  # noqa: F401
