"""openscene_b200: H100 (sm_90a) sparse-3D-convolution + open-vocabulary matching engine behind
OpenScene's MinkUNet (models/mink_unet.py) and run/evaluate.py.  See DESIGN.md."""
__all__ = ['me', 'coords', 'minkunet', 'synth']
