"""NumPy restatement of the training augmentation of ``dataset/augmentation.py`` and of the ``aug=True`` item chains of
``Point3DLoader`` (point_loader.py:156-174) and ``FusedFeatureLoader`` (feature_loader.py:102-189, train split).

It draws from the global ``random`` / ``np.random`` with the reference's calls, shapes and order, and spells out the
arithmetic the device kernels (csrc/augment.cu) must reproduce bit for bit:

* column min / max: ``(coords - min).max(0) == fl(max - min)`` because rounding is monotonic; float32 clouds stay
  float32 through ``// granularity`` (NumPy 2 treats Python scalars as weak).
* smoothing (scipy.ndimage.convolve, 3-tap box of float32(1/3), x then y then z, twice, mode='constant'): every output
  is accumulated in double from 0.0 over the taps at offsets -1, 0, +1, each tap ``double(x) * double(w)``, and rounded
  once to float32.
* interpolation (RegularGridInterpolator 'linear', scipy 1.18): the interval is the largest i <= n-2 with
  ``g[i] <= x``; ``y = (x - g[i]) / (g[i+1] - g[i])``; the 8 corners in ``itertools.product`` order, each weight
  ``((1 * w0) * w1) * w2`` with ``w = 1 - y`` (lower node) or ``y`` (upper node), each term ``double(v) * weight``,
  summed from ``0.`` corner by corner; out-of-bounds points get 0, NaN points NaN.  Then ``p + v * magnitude`` in
  float64.
* colours: float32 colours stay float32 through auto-contrast (weights rounded to float32); translation and jitter add
  in float64 and store back in the colour type; HSV runs in float64 and ends in the x86 uint8 cast (truncation to
  int32, low byte; NaN, inf and |x| >= 2^31 give 0).
"""
import itertools
import random

import numpy as np
import torch

from oracle import loader_ref, voxelize_ref

W3 = np.float64(np.float32(1) / np.float32(3))
ELASTIC_PARAMS = ((0.2, 0.4), (0.8, 1.6))


def blur(noise):
    g = np.asarray(noise, dtype=np.float32)
    for _ in range(2):
        for ax in range(3):
            a = g.astype(np.float64)
            n = a.shape[ax]
            lo, hi = np.zeros_like(a), np.zeros_like(a)
            sl = lambda s: tuple(s if d == ax else slice(None) for d in range(a.ndim))   # noqa: E731
            lo[sl(slice(1, n))] = a[sl(slice(0, n - 1))]
            hi[sl(slice(0, n - 1))] = a[sl(slice(1, n))]
            acc = 0.0 + lo * W3
            acc = acc + a * W3
            acc = acc + hi * W3
            g = acc.astype(np.float32)
    return g


def interp_add(coords, axes, noise, magnitude):
    p = np.asarray(coords).astype(np.float64)
    n = p.shape[0]
    idx, y = [], []
    oob = np.zeros(n, dtype=bool)
    nan = np.isnan(p).any(1)
    for d, g in enumerate(axes):
        g = np.asarray(g, dtype=np.float64)
        x = p[:, d]
        i = np.clip(np.searchsorted(g, x, side='right') - 1, 0, len(g) - 2)
        oob |= (x < g[0]) | (x > g[-1])
        idx.append(i)
        y.append((x - g[i]) / (g[i + 1] - g[i]))
    v = np.zeros((n, 3))
    for corner in itertools.product((0, 1), repeat=3):
        wt = np.ones(n)
        for d, h in enumerate(corner):
            wt = wt * (y[d] if h else 1 - y[d])
        vals = noise[idx[0] + corner[0], idx[1] + corner[1], idx[2] + corner[2]].astype(np.float64)
        v = v + vals * wt[:, None]
    v[oob] = 0.0
    v[nan] = np.nan
    return coords + v * magnitude


def elastic_grid(coords, granularity):
    """-> (coords_min, noise_dim) exactly as the reference derives them"""
    mn, mx = coords.min(0), coords.max(0)
    return mn, ((mx - mn) // granularity).astype(int) + 3


def elastic(coords, granularity, magnitude):
    mn, noise_dim = elastic_grid(coords, granularity)
    noise = blur(np.random.randn(*noise_dim, 3).astype(np.float32))
    axes = [np.linspace(lo, hi, d) for lo, hi, d in zip(mn - granularity, mn + granularity * (noise_dim - 2), noise_dim)]
    return interp_add(coords, axes, noise, magnitude)


def elastic_transform(coords, params=ELASTIC_PARAMS):
    if params is not None and random.random() < 0.95:
        for g, m in params:
            coords = elastic(coords, g, m)
    return coords


def u8(x):
    """x86 NumPy float64 -> uint8"""
    x = np.asarray(x, dtype=np.float64)
    ok = (x > -2147483649.0) & (x < 2147483648.0)
    t = np.where(ok, np.trunc(np.where(ok, x, 0.0)), 0.0).astype(np.int64)
    return (t & 255).astype(np.uint8)


def rem1(x):
    """np.remainder(x, 1.0) spelled out"""
    m = np.fmod(x, 1.0)
    return np.where(m == 0.0, 0.0, np.where(m < 0.0, m + 1.0, m))


def hsv_shift(rgb, hue, sat):
    """rgb_to_hsv, the hue / saturation translation and hsv_to_rgb, float64 until the uint8 cast."""
    rgb = np.asarray(rgb, dtype=np.float64)
    r, g, b = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    with np.errstate(invalid='ignore', divide='ignore'):
        nanrow = np.isnan(rgb).any(1)
        maxc = np.where(nanrow, np.nan, np.maximum(np.maximum(r, g), b))
        minc = np.where(nanrow, np.nan, np.minimum(np.minimum(r, g), b))
        mask = maxc != minc
        span = np.where(mask, maxc - minc, 1.0)
        s = np.where(mask, (maxc - minc) / np.where(mask, maxc, 1.0), 0.0)
        rc = np.where(mask, (maxc - r) / span, 0.0)
        gc = np.where(mask, (maxc - g) / span, 0.0)
        bc = np.where(mask, (maxc - b) / span, 0.0)
        h = np.where(r == maxc, bc - gc, np.where(g == maxc, (2.0 + rc) - bc, (4.0 + gc) - rc))
        h = rem1(h / 6.0)
        h = rem1((hue + h) + 1)
        s = np.clip(sat * s, 0, 1)
        h6 = h * 6.0
        i8 = u8(h6)
        f = h6 - i8
        v = maxc
        p, q, t = v * (1.0 - s), v * (1.0 - s * f), v * (1.0 - s * (1.0 - f))
        i = i8 % 6
        choice = np.where(s == 0.0, 6, i)          # 6: grey; np.select's first true condition wins
        table = {6: (v, v, v), 1: (q, v, p), 2: (p, v, t), 3: (p, q, v), 4: (t, p, v), 5: (v, p, q), 0: (v, t, p)}
        out = np.zeros((rgb.shape[0], 3))
        for k, (c0, c1, c2) in table.items():
            sel = choice == k
            out[sel, 0], out[sel, 1], out[sel, 2] = c0[sel], c1[sel], c2[sel]
    return u8(out)


def flip(coords):
    coords = coords.copy()
    if random.random() < 0.95:
        for ax in (0, 1):
            if random.random() < 0.5:
                coords[:, ax] = coords[:, ax].max() - coords[:, ax]
    return coords


def autocontrast(feats):
    if random.random() < 0.2:
        with np.errstate(invalid='ignore', divide='ignore'):
            lo, hi = feats.min(0), feats.max(0)
            cf = (feats - lo) * (255 / (hi - lo))
            b = random.random()
            feats = (1 - b) * feats + b * cf
    return feats


def translate(feats, ratio=0.1):
    feats = feats.copy()
    if random.random() < 0.95:
        tr = (np.random.rand(1, 3) - 0.5) * 255 * 2 * ratio
        feats[:, :3] = np.clip(feats[:, :3] + tr, 0, 255)
    return feats


def jitter(feats, std=0.05):
    feats = feats.copy()
    if random.random() < 0.95:
        noise = np.random.randn(feats.shape[0], 3) * (std * 255)
        feats[:, :3] = np.clip(feats[:, :3] + noise, 0, 255)
    return feats


def hue_sat(feats, hue_max=0.5, sat_max=0.2):
    feats = feats.copy()
    hue = (random.random() - 0.5) * 2 * hue_max
    sat = 1 + (random.random() - 0.5) * 2 * sat_max
    feats[:, :3] = hsv_shift(feats[:, :3], hue, sat)
    return feats


def input_transforms(coords, feats, trans_ratio=0.1, jitter_std=0.05, hue_max=0.5, sat_max=0.2):
    coords = flip(coords)
    feats = autocontrast(feats)
    feats = translate(feats, trans_ratio)
    feats = jitter(feats, jitter_std)
    return coords, hue_sat(feats, hue_max, sat_max)


def _finish(cv, feats, labels, batch_index, aug, input_color, **kw):
    if aug:
        cv, feats = input_transforms(cv, feats, **kw)
    coords = torch.from_numpy(cv).int()
    coords = torch.cat((torch.full((coords.shape[0], 1), batch_index, dtype=torch.int), coords), dim=1)
    feats = torch.from_numpy(feats).float() / 127.5 - 1. if input_color else torch.ones(coords.shape[0], 3)
    return coords, feats, torch.from_numpy(labels).long()


def point_item(locs_in, feats_in, labels_in, batch_index=0, voxel_size=0.05, aug=True, input_color=False, **kw):
    """Point3DLoader.__getitem__ from the transforms on, with the collate's batch column."""
    locs = elastic_transform(locs_in) if aug else locs_in
    M = voxelize_ref.transformation_matrix(voxel_size, np.random)
    cv, inds, _, _ = voxelize_ref.voxelize(locs, M)
    return _finish(cv, feats_in[inds], labels_in[inds], batch_index, aug, input_color, **kw)


def fused_item(locs_in, feats_in, labels_in, processed_data, batch_index=0, voxel_size=0.05, aug=True,
               input_color=False, **kw):
    """FusedFeatureLoader.__getitem__ on the train split: the distorted points are computed and dropped."""
    legacy = None
    if len(processed_data) > 2:
        legacy = torch.zeros(processed_data['feat'].shape[0], dtype=torch.bool)
        legacy[torch.as_tensor(processed_data['mask'])] = True
    if aug:
        elastic_transform(locs_in)
    M = voxelize_ref.transformation_matrix(voxel_size, np.random)
    cv, inds, _, _ = voxelize_ref.voxelize(locs_in, M)
    feat = torch.as_tensor(processed_data['feat'])
    feat = feat[..., 0] if feat.dim() > 2 else feat
    feat_3d, mask = loader_ref.remap_fused_features(feat, processed_data['mask_full'], inds, 'train', legacy_mask=legacy)
    coords, feats, labels = _finish(cv, feats_in[inds], labels_in[inds], batch_index, aug, input_color, **kw)
    return coords, feats, labels, feat_3d, mask
