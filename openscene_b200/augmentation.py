"""Training-time augmentation on the device (csrc/augment.cu), bit for bit with the reference's
``dataset/augmentation.py`` and the ``aug=True`` branches of ``Point3DLoader`` / ``FusedFeatureLoader``.

Every random draw stays on the host: the global ``random`` and ``np.random`` generators are consumed with the
reference's calls, shapes and order, so a training run draws the same stream whichever path builds its items.  What
moves to the GPU is the work that grows with the scene: the column min / max, the noise smoothing, the trilinear
interpolation over the points and one pass over the voxels for the flip and colour transforms.

* Drop-in classes (``ElasticDistortion``, ``RandomHorizontalFlip``, ``ChromaticAutoContrast``, ``ChromaticTranslation``,
  ``ChromaticJitter``, ``HueSaturationTranslation``, ``Compose``) keep the reference's constructors and ``__call__``
  signatures.  CUDA tensors in give CUDA tensors out; NumPy in gives NumPy out (computed on the device), as
  ``Voxelizer.voxelize`` does.  Results are new arrays; a gate that does not fire returns its inputs unchanged.
* ``DeviceItemAugmenter.point`` / ``.fused`` build one training item of ``Point3DLoader`` / ``FusedFeatureLoader``
  (``split='train'``) on the device, with at most three host synchronisations: the two elastic min / max reads and the
  voxel count.
"""
import ctypes
import random

import numpy as np
import torch

from . import _cabi as C
from .fused_features import remap_fused_features
from .voxelize import Voxelizer, voxelize_points

FLIP_X, FLIP_Y, AUTOCONTRAST, TRANSLATE, JITTER, HUE_SAT, INPUT_COLOR = 1, 2, 4, 8, 16, 32, 64
_DTYPE_CODE = {torch.float32: 0, torch.float64: 1, torch.int32: 2}


def _to_device(x, device='cuda'):
    """(CUDA tensor, came_from_numpy)"""
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x)).to(device), True
    C.require_cuda(x, 'input')
    return x.contiguous(), False


def _back(t, was_numpy):
    return t.cpu().numpy() if was_numpy else t


def _check_xyz(t, what):
    if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] == 0:
        raise ValueError(f"{what}: expected a non-empty [N, 3] array, got shape {tuple(t.shape)}")
    if t.dtype not in _DTYPE_CODE:
        raise TypeError(f"{what}: dtype {t.dtype} is not float32, float64 or int32")


def column_minmax(x, rows=None):
    """[2c] float64 CUDA tensor: column minima then maxima of x [N, c] (of x[rows] when rows is given).  No sync."""
    if x.dtype not in _DTYPE_CODE:
        raise TypeError(f"column_minmax: dtype {x.dtype} is not float32, float64 or int32")
    x = x.contiguous()
    c = x.shape[1]
    n = rows.numel() if rows is not None else x.shape[0]
    dev = x.device
    with torch.cuda.device(dev):
        ws_bytes = C.lib().osb_aug_minmax_workspace_bytes(c)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        out = torch.empty(2 * c, dtype=torch.float64, device=dev)
        C.call('osb_aug_minmax', C.ptr(x), _DTYPE_CODE[x.dtype], C.ptr(rows), n, c, C.ptr(out), C.ptr(ws), ws_bytes,
               C.stream_ptr())
    return out


def blur_noise(noise):
    """ElasticDistortion's smoothing (augmentation.py:171-184) of a float32 [X, Y, Z, ch] CUDA grid, in place."""
    assert noise.dtype == torch.float32 and noise.dim() == 4 and noise.is_contiguous()
    X, Y, Z, ch = noise.shape
    with torch.cuda.device(noise.device):
        tmp = torch.empty_like(noise)
        C.call('osb_aug_blur', C.ptr(noise), C.ptr(tmp), X, Y, Z, ch, C.stream_ptr())
    return noise


def elastic_interp(pts, axes, noise, magnitude):
    """pts + RegularGridInterpolator(axes, noise, bounds_error=0, fill_value=0)(pts) * magnitude, float64 [N, 3]."""
    _check_xyz(pts, 'elastic_interp')
    if pts.dtype == torch.int32:
        raise TypeError("elastic_interp: points must be float32 or float64")
    dims = [len(a) for a in axes]
    assert tuple(noise.shape) == (*dims, 3) and noise.dtype == torch.float32
    dev = pts.device
    with torch.cuda.device(dev):
        ax = torch.from_numpy(np.concatenate([np.asarray(a, dtype=np.float64) for a in axes])).to(dev)
        out = torch.empty((pts.shape[0], 3), dtype=torch.float64, device=dev)
        C.call('osb_aug_elastic_interp', C.ptr(pts), int(pts.dtype == torch.float64), pts.shape[0], C.ptr(noise),
               dims[0], dims[1], dims[2], C.ptr(ax), float(magnitude), C.ptr(out), C.stream_ptr())
    return out


def elastic_distortion(pts, granularity, magnitude, interpolate=True):
    """``ElasticDistortion.elastic_distortion`` for a CUDA [N, 3] float tensor (one host sync, for the min / max).
    The noise is drawn with ``np.random.randn`` exactly as the reference draws it.  interpolate=False consumes the
    draw and returns None (the fused-feature loader discards the distorted points)."""
    np_dtype = np.float32 if pts.dtype == torch.float32 else np.float64
    mm = column_minmax(pts).cpu().numpy()
    if not np.all(np.isfinite(mm)):
        raise ValueError("ElasticDistortion: non-finite coordinates")
    coords_min, coords_max = mm[:3].astype(np_dtype), mm[3:].astype(np_dtype)
    # (coords - min).max(0) == fl(max - min): rounding is monotonic; the rest is the reference's host arithmetic
    noise_dim = ((coords_max - coords_min) // granularity).astype(int) + 3
    noise = np.random.randn(*noise_dim, 3).astype(np.float32)
    if not interpolate:
        return None
    ax = [np.linspace(d_min, d_max, d)
          for d_min, d_max, d in zip(coords_min - granularity, coords_min + granularity * (noise_dim - 2), noise_dim)]
    grid = blur_noise(torch.from_numpy(noise).to(pts.device))
    return elastic_interp(pts, ax, grid, magnitude)


def _input_pass(coords, feats, stages, params, jitter=None, labels=None, rows=None, batch_index=0, item=False,
                generic=True):
    """One launch of osb_aug_input_transforms.  generic: return (coords, feats) in their own types; item: return the
    loader's (coords int32 [n,4], feats float32 [n,3], labels int64 [n])."""
    if feats.dim() != 2 or feats.shape[1] != 3:
        raise ValueError(f"only 3-column colours are supported, got shape {tuple(feats.shape)}")
    if feats.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"colours must be float32 or float64, got {feats.dtype}")
    _check_xyz(coords, 'coords')
    n = coords.shape[0]
    if rows is None and feats.shape[0] != n:
        raise ValueError("coords and feats have different row counts")
    dev = coords.device
    with torch.cuda.device(dev):
        cmax = column_minmax(coords)[3:] if stages & (FLIP_X | FLIP_Y) else None
        fmm = column_minmax(feats, rows) if stages & AUTOCONTRAST else None
        if jitter is not None:
            jitter = torch.from_numpy(np.ascontiguousarray(jitter, dtype=np.float64)).to(dev)
        p = np.ascontiguousarray(params, dtype=np.float64)
        c_out = torch.empty_like(coords) if generic else None
        f_out = torch.empty((n, 3), dtype=feats.dtype, device=dev) if generic else None
        ic = torch.empty((n, 4), dtype=torch.int32, device=dev) if item else None
        if_ = torch.empty((n, 3), dtype=torch.float32, device=dev) if item else None
        il = torch.empty(n, dtype=torch.int64, device=dev) if item else None
        C.call('osb_aug_input_transforms', C.ptr(coords), _DTYPE_CODE[coords.dtype], C.ptr(feats),
               int(feats.dtype == torch.float64), C.ptr(labels), C.ptr(rows), n, C.ptr(cmax), C.ptr(fmm), C.ptr(jitter),
               p.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), stages, int(batch_index), C.ptr(c_out), C.ptr(f_out),
               C.ptr(ic), C.ptr(if_), C.ptr(il), C.stream_ptr())
    return (ic, if_, il) if item else (c_out, f_out)


def _draw_input_transforms(n, trans_ratio, jitter_std, hue_max, sat_max):
    """The host draws of the loaders' five input transforms, in the reference's order.  -> (stages, params, jitter)"""
    stages, params, jitter = 0, np.zeros(8), None
    if random.random() < 0.95:                                  # RandomHorizontalFlip('z'): axes 0 then 1
        for ax in (0, 1):
            if random.random() < 0.5:
                stages |= FLIP_X << ax
    if random.random() < 0.2:                                   # ChromaticAutoContrast
        b = random.random()
        params[0], params[1] = 1 - b, b
        stages |= AUTOCONTRAST
    if random.random() < 0.95:                                  # ChromaticTranslation
        params[2:5] = ((np.random.rand(1, 3) - 0.5) * 255 * 2 * trans_ratio)[0]
        stages |= TRANSLATE
    if random.random() < 0.95:                                  # ChromaticJitter
        jitter = np.random.randn(n, 3)
        params[5] = jitter_std * 255
        stages |= JITTER
    params[6] = (random.random() - 0.5) * 2 * hue_max           # HueSaturationTranslation
    params[7] = 1 + (random.random() - 0.5) * 2 * sat_max
    return stages | HUE_SAT, params, jitter


# ----------------------------------------------------------------------------------------- drop-in transform classes
class ChromaticTranslation:
    def __init__(self, trans_range_ratio=1e-1):
        self.trans_range_ratio = trans_range_ratio

    def __call__(self, coords, feats, labels):
        if random.random() < 0.95:
            tr = (np.random.rand(1, 3) - 0.5) * 255 * 2 * self.trans_range_ratio
            feats = _single(coords, feats, TRANSLATE, {2: tr[0]})
        return coords, feats, labels


class ChromaticAutoContrast:
    def __init__(self, randomize_blend_factor=True, blend_factor=0.5):
        self.randomize_blend_factor = randomize_blend_factor
        self.blend_factor = blend_factor

    def __call__(self, coords, feats, labels):
        if random.random() < 0.2:
            b = random.random() if self.randomize_blend_factor else self.blend_factor
            feats = _single(coords, feats, AUTOCONTRAST, {0: [1 - b, b]})
        return coords, feats, labels


class ChromaticJitter:
    def __init__(self, std=0.01):
        self.std = std

    def __call__(self, coords, feats, labels):
        if random.random() < 0.95:
            noise = np.random.randn(feats.shape[0], 3)
            feats = _single(coords, feats, JITTER, {5: [self.std * 255]}, jitter=noise)
        return coords, feats, labels


class HueSaturationTranslation:
    def __init__(self, hue_max, saturation_max):
        self.hue_max = hue_max
        self.saturation_max = saturation_max

    def __call__(self, coords, feats, labels):
        hue_val = (random.random() - 0.5) * 2 * self.hue_max
        sat_ratio = 1 + (random.random() - 0.5) * 2 * self.saturation_max
        feats = _single(coords, feats, HUE_SAT, {6: [hue_val, sat_ratio]})
        return coords, feats, labels


class RandomHorizontalFlip:
    def __init__(self, upright_axis, is_temporal):
        self.is_temporal = is_temporal
        self.D = 4 if is_temporal else 3
        self.upright_axis = {'x': 0, 'y': 1, 'z': 2}[upright_axis.lower()]
        self.horz_axes = set(range(self.D)) - set([self.upright_axis])
        if self.D != 3:
            raise NotImplementedError("temporal (4-D) coordinates are not used by any OpenScene loader")

    def __call__(self, coords, feats, labels):
        if random.random() < 0.95:
            stages = 0
            for curr_ax in self.horz_axes:
                if random.random() < 0.5:
                    stages |= 1 << curr_ax
            if stages:
                c, was_np = _to_device(coords)
                _check_xyz(c, 'RandomHorizontalFlip')
                if stages & 4:                                   # a flip of axis 2: rotate the axes into slots 0 / 1
                    perm = [a for a in range(3) if a != self.upright_axis] + [self.upright_axis]
                    inv = [perm.index(a) for a in range(3)]
                    cp = c[:, perm].contiguous()
                    s = sum(1 << perm.index(a) for a in range(3) if stages >> a & 1)
                    out = _input_pass(cp, _dummy_feats(cp), s, np.zeros(8))[0][:, inv].contiguous()
                else:
                    out = _input_pass(c, _dummy_feats(c), stages, np.zeros(8))[0]
                coords = _back(out, was_np)
        return coords, feats, labels


class ElasticDistortion:
    def __init__(self, distortion_params):
        self.distortion_params = distortion_params

    def elastic_distortion(self, coords, granularity, magnitude):
        c, was_np = _to_device(coords)
        _check_xyz(c, 'ElasticDistortion')
        return _back(elastic_distortion(c, granularity, magnitude), was_np)

    def __call__(self, pointcloud):
        if self.distortion_params is not None:
            if random.random() < 0.95:
                c, was_np = _to_device(pointcloud)
                _check_xyz(c, 'ElasticDistortion')
                for granularity, magnitude in self.distortion_params:
                    c = elastic_distortion(c, granularity, magnitude)
                pointcloud = _back(c, was_np)
        return pointcloud


class Compose:
    def __init__(self, transforms):
        self.transforms = transforms

    def __call__(self, *args):
        for t in self.transforms:
            args = t(*args)
        return args


def _dummy_feats(c):
    return torch.zeros((c.shape[0], 3), dtype=torch.float32, device=c.device)


def _single(coords, feats, stage, set_params, jitter=None):
    """One colour transform on the device; NumPy in -> NumPy out."""
    f, was_np = _to_device(feats)
    params = np.zeros(8)
    for k, v in set_params.items():
        params[k:k + len(v)] = v
    xyz = torch.zeros((f.shape[0], 3), dtype=torch.int32, device=f.device) if f.dim() == 2 else f
    out = _input_pass(xyz, f, stage, params, jitter=jitter)[1]
    return _back(out, was_np)


# ----------------------------------------------------------------------------------------- per-item device path
class DeviceItemAugmenter:
    """Builds the training items of ``Point3DLoader`` / ``FusedFeatureLoader`` (``split='train'``, ``eval_all=False``)
    on the device from what their workers load.  The constants are the loaders' class attributes
    (``dataset/point_loader.py:58-66``) and ``__init__`` arguments."""
    SCALE_AUGMENTATION_BOUND = (0.9, 1.1)
    ROTATION_AUGMENTATION_BOUND = ((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi))
    TRANSLATION_AUGMENTATION_RATIO_BOUND = ((-0.2, 0.2), (-0.2, 0.2), (0, 0))
    ELASTIC_DISTORT_PARAMS = ((0.2, 0.4), (0.8, 1.6))

    def __init__(self, voxel_size=0.05, aug=True, input_color=False, data_aug_color_trans_ratio=0.1,
                 data_aug_color_jitter_std=0.05, data_aug_hue_max=0.5, data_aug_saturation_max=0.2, device='cuda'):
        self.aug, self.input_color, self.device = aug, input_color, torch.device(device)
        self.trans_ratio, self.jitter_std = data_aug_color_trans_ratio, data_aug_color_jitter_std
        self.hue_max, self.sat_max = data_aug_hue_max, data_aug_saturation_max
        self.voxelizer = Voxelizer(voxel_size=voxel_size, clip_bound=None, use_augmentation=True,
                                   scale_augmentation_bound=self.SCALE_AUGMENTATION_BOUND,
                                   rotation_augmentation_bound=self.ROTATION_AUGMENTATION_BOUND,
                                   translation_augmentation_ratio_bound=self.TRANSLATION_AUGMENTATION_RATIO_BOUND)

    def _load(self, locs_in, feats_in, labels_in):
        locs = torch.as_tensor(locs_in).to(self.device).contiguous()
        feats = torch.as_tensor(feats_in).to(self.device).contiguous()
        labels = torch.as_tensor(labels_in).to(self.device).to(torch.uint8).contiguous()
        _check_xyz(locs, 'locs')
        if locs.dtype == torch.int32:
            raise TypeError("locs must be float32 or float64")
        if feats.shape != locs.shape or feats.dtype not in (torch.float32, torch.float64):
            raise ValueError(f"feats must be float32 / float64 [N, 3] like locs, got {feats.dtype} {tuple(feats.shape)}")
        if labels.shape != (locs.shape[0],):
            raise ValueError("labels must have one entry per point")
        return locs, feats, labels

    def _elastic(self, locs, interpolate=True):
        if random.random() < 0.95:
            params = self.ELASTIC_DISTORT_PARAMS
            for k, (granularity, magnitude) in enumerate(params):
                last = k == len(params) - 1
                out = elastic_distortion(locs, granularity, magnitude, interpolate=interpolate or not last)
                locs = out if out is not None else locs
        return locs

    def _voxelize(self, locs):
        M_v, M_r = self.voxelizer.get_transformation_matrix()
        cv, inds, _, _ = voxelize_points(locs, M_r @ M_v)
        return cv, inds

    def _finish(self, cv, feats, labels, inds, batch_index):
        if self.aug:
            stages, params, jitter = _draw_input_transforms(cv.shape[0], self.trans_ratio, self.jitter_std, self.hue_max,
                                                            self.sat_max)
        else:
            stages, params, jitter = 0, np.zeros(8), None
        if self.input_color:
            stages |= INPUT_COLOR
        return _input_pass(cv, feats, stages, params, jitter=jitter, labels=labels, rows=inds, batch_index=batch_index,
                           item=True, generic=False)

    def point(self, locs_in, feats_in, labels_in, batch_index=0):
        """``Point3DLoader.__getitem__`` from the transforms on (point_loader.py:156-174), with the collate's batch
        column: -> CUDA (coords int32 [Nv,4], feats float32 [Nv,3], labels int64 [Nv])."""
        locs, feats, labels = self._load(locs_in, feats_in, labels_in)
        if self.aug:
            locs = self._elastic(locs)
        cv, inds = self._voxelize(locs)
        return self._finish(cv, feats, labels, inds, batch_index)

    def fused(self, locs_in, feats_in, labels_in, processed_data, batch_index=0):
        """``FusedFeatureLoader.__getitem__`` on the train split (feature_loader.py:102-189): -> CUDA (coords, feats,
        labels, feat_3d, mask).  The reference distorts the points and then voxelises ``locs_in``, so the elastic
        draws are consumed (the first pass still runs: its output sizes the second draw) and the distortion is
        dropped, as there."""
        locs, feats, labels = self._load(locs_in, feats_in, labels_in)
        keys = list(processed_data.keys())
        feat_3d, mask_full = processed_data['feat'], processed_data['mask_full']
        legacy = None
        if len(keys) > 2:                                        # the old three-key files (:114-117)
            legacy = torch.zeros(feat_3d.shape[0], dtype=torch.bool)
            legacy[torch.as_tensor(processed_data['mask'])] = True
        if self.aug:
            self._elastic(locs, interpolate=False)
        cv, inds = self._voxelize(locs)
        feat_vox, mask = remap_fused_features(feat_3d, mask_full, inds, 'train', legacy_mask=legacy, device=self.device)
        coords, feats_o, labels_o = self._finish(cv, feats, labels, inds, batch_index)
        return coords, feats_o, labels_o, feat_vox, mask
