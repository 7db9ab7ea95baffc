"""The NumPy augmentation oracle (tests/augment_ref.py) against the reference's own outputs, bit for bit and draw for draw:
the committed goldens always, and the reference's classes live where the reference tree exists."""
import os
import random
import sys

import numpy as np
import pytest
import scipy.interpolate
import scipy.ndimage
import torch

from tests import augment_ref as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF = '/root/reference'


def same(a, b):
    """equal dtype, shape and bits (NaN payloads included)"""
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def golden(name):
    z = np.load(os.path.join(GOLDEN, f'augment_{name}.npz'))
    cases = []
    for k in range(int(z['n'])):
        pre = f'c{k}_'
        c = {'seed': int(z[pre + 'seed']), 'in': {}, 'out': {}, 'next_py': z[pre + 'next_py'], 'next_np': z[pre + 'next_np']}
        for key in z.files:
            if key.startswith(pre + 'in_'):
                c['in'][key[len(pre) + 3:]] = z[key]
            elif key.startswith(pre + 'out_'):
                c['out'][key[len(pre) + 4:]] = z[key]
        if 'kinds' in z.files:
            c['kind'] = str(z['kinds'][k])
        cases.append(c)
    return cases


def seed(s):
    random.seed(s)
    np.random.seed(s)


def next_draws():
    return np.array([random.random() for _ in range(3)]), np.random.rand(3)


def check_draws(case):
    py, npr = next_draws()
    assert same(py, case['next_py']) and same(npr, case['next_np']), "the generators were consumed differently"


ORACLE_COLOUR = {
    'flip': lambda c, f: (A.flip(c), f),
    'autocontrast': lambda c, f: (c, A.autocontrast(f)),
    'translation': lambda c, f: (c, A.translate(f, 0.1)),
    'jitter': lambda c, f: (c, A.jitter(f, 0.05)),
    'hue_sat': lambda c, f: (c, A.hue_sat(f, 0.5, 0.2)),
    'chain': lambda c, f: A.input_transforms(c, f),
}


@pytest.mark.parametrize('k', range(7))
def test_oracle_elastic_equals_golden(k):
    case = golden('elastic')[k]
    seed(case['seed'])
    params = None if k == 6 else A.ELASTIC_PARAMS
    out = A.elastic_transform(case['in']['pointcloud'].copy(), params)
    assert same(out, case['out']['coords'])
    check_draws(case)


@pytest.mark.parametrize('k', range(26))
def test_oracle_colour_transforms_equal_golden(k):
    case = golden('colour')[k]
    seed(case['seed'])
    with np.errstate(invalid='ignore', divide='ignore'):
        c, f = ORACLE_COLOUR[case['kind']](case['in']['coords'].copy(), case['in']['feats'].copy())
    assert same(c, case['out']['coords']), case['kind']
    assert same(f, case['out']['feats']), case['kind']
    check_draws(case)


@pytest.mark.parametrize('kind', ['point', 'fused'])
@pytest.mark.parametrize('k', range(5))
def test_oracle_items_equal_golden(kind, k):
    case = golden(kind)[k]
    i = case['in']
    seed(case['seed'])
    with np.errstate(invalid='ignore', divide='ignore'):
        if kind == 'point':
            out = A.point_item(i['locs'], i['feats'], i['labels'], batch_index=1, input_color=bool(i['input_color']))
            names = ('coords', 'feats', 'labels')
        else:
            blob = {'feat': torch.from_numpy(i['feat']), 'mask_full': torch.from_numpy(i['mask_full'])}
            out = A.fused_item(i['locs'], i['feats'], i['labels'], blob, batch_index=1, input_color=bool(i['input_color']))
            names = ('coords', 'feats', 'labels', 'feat_3d', 'mask')
    for nm, o in zip(names, out):
        assert same(o.numpy(), case['out'][nm]), nm
    check_draws(case)


def test_golden_covers_the_edges():
    colour = golden('colour')
    kinds = [c['kind'] for c in colour]
    for kind in ('flip', 'autocontrast', 'translation', 'jitter', 'hue_sat', 'chain'):
        assert kind in kinds
    # the constant-colour chain: auto-contrast divided by zero and the HSV cast turned the NaN into 0
    const = [c for c in colour if c['kind'] == 'chain']
    assert all(np.all(c['out']['feats'] == 0) for c in const)
    # gates both ways: unchanged outputs exist for every gated transform
    for kind in ('flip', 'autocontrast', 'translation', 'jitter'):
        cs = [c for c in colour if c['kind'] == kind]
        assert any(same(c['out']['feats'], c['in']['feats']) and same(c['out']['coords'], c['in']['coords']) for c in cs)
        assert any(not (same(c['out']['feats'], c['in']['feats']) and same(c['out']['coords'], c['in']['coords'])) for c in cs)
    el = golden('elastic')
    assert any(same(c['out']['coords'], c['in']['pointcloud']) for c in el)
    assert {c['in']['pointcloud'].dtype for c in el} == {np.dtype(np.float32), np.dtype(np.float64)}
    assert {len(c['in']['pointcloud']) for c in el} >= {1, 2}


def test_u8_cast_is_the_x86_numpy_cast():
    x = np.array([np.nan, np.inf, -np.inf, -1.5, -0.3, 0.0, 0.7, 255.9, 256.0, 300.7, -300.2, 65543.5, 2147483647.9,
                  2147483648.0, -2147483648.9, -2147483649.0, 5e9, 1e300])
    with np.errstate(invalid='ignore'):
        assert same(A.u8(x), x.astype('uint8'))


def test_blur_equals_scipy_on_random_grids():
    rng = np.random.default_rng(3)
    for shape in [(3, 3, 3), (5, 9, 4), (17, 11, 6), (1, 4, 2)]:
        big = rng.choice([-1, 1], (*shape, 3)) * 2.0 ** rng.integers(10, 40, (*shape, 3))
        x = np.where(rng.random((*shape, 3)) < 0.5, big, rng.standard_normal((*shape, 3))).astype(np.float32)
        ref = x
        for _ in range(2):
            for kshape in ((3, 1, 1, 1), (1, 3, 1, 1), (1, 1, 3, 1)):
                ref = scipy.ndimage.convolve(ref, np.ones(kshape).astype('float32') / 3, mode='constant', cval=0)
        assert same(A.blur(x), ref), shape


def test_interpolation_equals_scipy_on_random_grids():
    rng = np.random.default_rng(4)
    for dims in [(3, 3, 3), (7, 5, 4), (20, 13, 9)]:
        mn = rng.standard_normal(3)
        g = rng.uniform(0.05, 1.0)
        axes = [np.linspace(mn[d] - g, mn[d] + g * (dims[d] - 2), dims[d]) for d in range(3)]
        noise = rng.standard_normal((*dims, 3)).astype(np.float32)
        span = [(a[0] - 0.3 * g, a[-1] + 0.3 * g) for a in axes]
        pts = np.stack([rng.uniform(*span[d], 4000) for d in range(3)], 1)
        nodes = np.stack([rng.choice(axes[d], 500) for d in range(3)], 1)          # exactly on grid nodes and edges
        pts = np.concatenate([pts, nodes, [[a[-1] for a in axes], [a[0] for a in axes]]])
        for dt in (np.float32, np.float64):
            p = pts.astype(dt)
            ref = p + scipy.interpolate.RegularGridInterpolator(axes, noise, bounds_error=0, fill_value=0)(p) * 0.4
            assert same(A.interp_add(p, axes, noise, 0.4), ref)


# ------------------------------------------------------------------------------------------- live, against the reference
def _reference():
    if not os.path.isdir(os.path.join(REF, 'dataset')):
        pytest.skip('reference tree not available')
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import dataset.augmentation as t
    return t


@pytest.mark.parametrize('case', range(30))
def test_oracle_equals_reference_live(case):
    t = _reference()
    rng = np.random.RandomState(900 + case)
    dt = np.float32 if case % 2 else np.float64
    n = [1, 2, 3, 50, 700, 3000][case % 6]
    pts = (rng.rand(n, 3) * rng.uniform(0.1, 4.0, 3) + rng.uniform(-3, 3, 3)).astype(dt)
    feats = (rng.rand(n, 3) * 255).astype(dt)
    if case % 5 == 0:
        feats[:, case % 3] = feats[0, case % 3]                                   # a constant colour column
    if case % 7 == 0:
        feats[:] = 127.5
    coords = np.floor(rng.rand(n, 3) * 30)
    labels = np.arange(n)
    chain = t.Compose([t.RandomHorizontalFlip('z', False), t.ChromaticAutoContrast(), t.ChromaticTranslation(0.1),
                       t.ChromaticJitter(0.05), t.HueSaturationTranslation(0.5, 0.2)])
    s = 5000 + case
    seed(s)
    ref_pts = t.ElasticDistortion(A.ELASTIC_PARAMS)(pts.copy())
    with np.errstate(invalid='ignore', divide='ignore'):
        ref_c, ref_f, _ = chain(coords.copy(), feats.copy(), labels.copy())
    ref_next = next_draws()
    seed(s)
    got_pts = A.elastic_transform(pts.copy())
    with np.errstate(invalid='ignore', divide='ignore'):
        got_c, got_f = A.input_transforms(coords.copy(), feats.copy())
    assert same(got_pts, ref_pts) and same(got_c, ref_c) and same(got_f, ref_f)
    got_next = next_draws()
    assert same(got_next[0], ref_next[0]) and same(got_next[1], ref_next[1])
