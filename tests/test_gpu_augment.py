"""Device augmentation (openscene_b200/augmentation.py, csrc/augment.cu) against the reference's outputs and the NumPy
oracle, bit for bit and draw for draw."""
import ctypes
import random

import numpy as np
import pytest
import scipy.interpolate
import scipy.ndimage
import torch

from tests import augment_ref as A
from tests.test_augment_ref_cpu import ORACLE_COLOUR, check_draws, golden, next_draws, same, seed

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _aug():
    from openscene_b200 import augmentation
    return augmentation


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _product_colour(kind):
    aug = _aug()
    tf = {'flip': aug.RandomHorizontalFlip('z', False), 'autocontrast': aug.ChromaticAutoContrast(),
          'translation': aug.ChromaticTranslation(0.1), 'jitter': aug.ChromaticJitter(0.05),
          'hue_sat': aug.HueSaturationTranslation(0.5, 0.2)}
    if kind == 'chain':
        return aug.Compose([tf[k] for k in ('flip', 'autocontrast', 'translation', 'jitter', 'hue_sat')])
    return tf[kind]


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize('k', range(7))
@pytest.mark.parametrize('where', ['numpy', 'cuda'])
def test_elastic_equals_golden(k, where):
    aug = _aug()
    case = golden('elastic')[k]
    pc = case['in']['pointcloud'].copy()
    if where == 'cuda':
        pc = torch.from_numpy(pc).to(DEV)
    seed(case['seed'])
    out = aug.ElasticDistortion(None if k == 6 else A.ELASTIC_PARAMS)(pc)
    assert isinstance(out, np.ndarray) == (where == 'numpy')
    assert same(_np(out), case['out']['coords'])
    check_draws(case)


@pytest.mark.parametrize('k', range(26))
@pytest.mark.parametrize('where', ['numpy', 'cuda'])
def test_colour_transforms_equal_golden(k, where):
    case = golden('colour')[k]
    c, f, lab = case['in']['coords'].copy(), case['in']['feats'].copy(), case['in']['labels'].copy()
    if where == 'cuda':
        c, f = torch.from_numpy(c).to(DEV), torch.from_numpy(f).to(DEV)
    seed(case['seed'])
    oc, of, ol = _product_colour(case['kind'])(c, f, lab)
    assert same(_np(oc), case['out']['coords']) and same(_np(of), case['out']['feats']), case['kind']
    assert ol is lab
    check_draws(case)


def _item(kind, i, batch_index):
    aug = _aug()
    it = aug.DeviceItemAugmenter(voxel_size=0.05, input_color=bool(i['input_color']))
    if kind == 'point':
        return it.point(i['locs'], i['feats'], i['labels'], batch_index=batch_index)
    blob = {'feat': torch.from_numpy(i['feat']), 'mask_full': torch.from_numpy(i['mask_full'])}
    return it.fused(i['locs'], i['feats'], i['labels'], blob, batch_index=batch_index)


@pytest.mark.parametrize('kind', ['point', 'fused'])
@pytest.mark.parametrize('k', range(5))
def test_items_equal_golden(kind, k):
    case = golden(kind)[k]
    seed(case['seed'])
    out = _item(kind, case['in'], 1)
    names = ('coords', 'feats', 'labels', 'feat_3d', 'mask')
    for nm, o in zip(names, out):
        assert o.is_cuda
        assert same(o.cpu().numpy(), case['out'][nm]), nm
    check_draws(case)


# ------------------------------------------------------------------------------------------------ live against the oracle
def _cloud(name):
    from openscene_b200 import synth
    if name.startswith('lidar'):
        pts = synth.lidar_points(60_000, seed=3)
    elif name.startswith('tiny'):
        pts = np.random.RandomState(int(name[-1])).rand(int(name[-1]), 3) * 3
    else:
        pts, _ = synth.scene_points(name, seed=1)
    return pts


@pytest.mark.parametrize('name,dt,color', [('tiny1', np.float32, True), ('tiny2', np.float64, True),
                                           ('config1_50k', np.float32, False), ('config1_50k', np.float64, True),
                                           ('config2_200k', np.float32, True), ('lidar', np.float64, True)])
@pytest.mark.parametrize('kind', ['point', 'fused'])
def test_items_equal_oracle_live(name, dt, color, kind):
    pts = _cloud(name).astype(dt)
    n = len(pts)
    rng = np.random.RandomState(n % 1000)
    colors = (rng.rand(n, 3) * 2 - 1).astype(dt)
    feats = (colors + 1.) * 127.5
    labels = rng.randint(0, 21, n).astype(np.uint8)
    mask_full = rng.rand(n) < 0.6
    mask_full[0] = True
    feat = rng.randn(int(mask_full.sum()), 16).astype(np.float16)
    blob = {'feat': torch.from_numpy(feat), 'mask_full': torch.from_numpy(mask_full)}
    i = dict(locs=pts, feats=feats, labels=labels, feat=feat, mask_full=mask_full, input_color=color)
    for s in (11, _seed_skipping_elastic()):
        seed(s)
        with np.errstate(invalid='ignore', divide='ignore'):
            if kind == 'point':
                ref = A.point_item(pts, feats, labels, batch_index=3, input_color=color)
            else:
                ref = A.fused_item(pts, feats, labels, blob, batch_index=3, input_color=color)
        ref_next = next_draws()
        seed(s)
        got = _item(kind, i, 3)
        got_next = next_draws()
        for r, g in zip(ref, got):
            assert same(g.cpu().numpy(), r.numpy())
        assert same(got_next[0], ref_next[0]) and same(got_next[1], ref_next[1])


def _seed_skipping_elastic():
    s = 0
    while random.Random(s).random() < 0.95:
        s += 1
    return s


def test_two_runs_are_bit_identical():
    pts, _ = _cloud('config1_50k'), None
    n = len(pts)
    feats = np.random.RandomState(0).rand(n, 3) * 255
    labels = np.zeros(n, dtype=np.uint8)
    i = dict(locs=pts, feats=feats, labels=labels, input_color=True)
    outs = []
    for _ in range(2):
        seed(5)
        outs.append([o.cpu().numpy() for o in _item('point', i, 0)])
    for a, b in zip(*outs):
        assert same(a, b)


# ------------------------------------------------------------------------------------------------ kernels vs scipy itself
def test_blur_equals_scipy():
    aug = _aug()
    rng = np.random.default_rng(7)
    for shape in [(3, 3, 3), (1, 5, 2), (23, 17, 9), (61, 40, 22)]:
        big = rng.choice([-1, 1], (*shape, 3)) * 2.0 ** rng.integers(10, 40, (*shape, 3))
        x = np.where(rng.random((*shape, 3)) < 0.5, big, rng.standard_normal((*shape, 3))).astype(np.float32)
        ref = x
        for _ in range(2):
            for kshape in ((3, 1, 1, 1), (1, 3, 1, 1), (1, 1, 3, 1)):
                ref = scipy.ndimage.convolve(ref, np.ones(kshape).astype('float32') / 3, mode='constant', cval=0)
        got = aug.blur_noise(torch.from_numpy(x).to(DEV)).cpu().numpy()
        assert same(got, ref), shape


def test_interpolation_equals_scipy():
    aug = _aug()
    rng = np.random.default_rng(8)
    for dims in [(3, 3, 3), (9, 6, 4), (40, 30, 12)]:
        mn, g = rng.standard_normal(3), rng.uniform(0.05, 1.0)
        axes = [np.linspace(mn[d] - g, mn[d] + g * (dims[d] - 2), dims[d]) for d in range(3)]
        noise = rng.standard_normal((*dims, 3)).astype(np.float32)
        span = [(a[0] - 0.3 * g, a[-1] + 0.3 * g) for a in axes]
        pts = np.stack([rng.uniform(*span[d], 20000) for d in range(3)], 1)
        nodes = np.stack([rng.choice(axes[d], 2000) for d in range(3)], 1)
        pts = np.concatenate([pts, nodes, [[a[-1] for a in axes], [a[0] for a in axes]]])
        for dt in (np.float32, np.float64):
            p = pts.astype(dt)
            ref = p + scipy.interpolate.RegularGridInterpolator(axes, noise, bounds_error=0, fill_value=0)(p) * 1.6
            got = aug.elastic_interp(torch.from_numpy(p).to(DEV), axes, torch.from_numpy(noise).to(DEV), 1.6)
            assert same(got.cpu().numpy(), ref)


def test_entry_points_write_every_output_into_nan_filled_buffers():
    """the C entry points on NaN-prefilled outputs: every element is written, and equals the oracle"""
    from openscene_b200 import _cabi as C
    rng = np.random.default_rng(9)
    n = 70_001
    pts = torch.from_numpy(rng.uniform(-1, 3, (n, 3))).to(DEV)
    dims = (9, 7, 5)
    axes = [np.linspace(-1.2, 3.2, d) for d in dims]
    noise = rng.standard_normal((*dims, 3)).astype(np.float32)
    ax = torch.from_numpy(np.concatenate(axes)).to(DEV)
    nz = torch.from_numpy(noise).to(DEV)
    out = torch.full((n, 3), float('nan'), dtype=torch.float64, device=DEV)
    C.call('osb_aug_elastic_interp', C.ptr(pts), 1, n, C.ptr(nz), *dims, C.ptr(ax), 0.4, C.ptr(out), C.stream_ptr())
    assert same(out.cpu().numpy(), A.interp_add(pts.cpu().numpy(), axes, noise, 0.4))
    mm = torch.full((6,), float('nan'), dtype=torch.float64, device=DEV)
    ws = torch.empty(C.lib().osb_aug_minmax_workspace_bytes(3), dtype=torch.uint8, device=DEV)
    C.call('osb_aug_minmax', C.ptr(pts), 1, None, n, 3, C.ptr(mm), C.ptr(ws), ws.numel(), C.stream_ptr())
    p = pts.cpu().numpy()
    assert same(mm.cpu().numpy(), np.concatenate([p.min(0), p.max(0)]))
    # one voxel pass with every stage on, item outputs prefilled with NaN / sentinels
    cv = torch.from_numpy(rng.integers(0, 500, (n, 3)).astype(np.int32)).to(DEV)
    f32 = torch.from_numpy((rng.random((n, 3)) * 255).astype(np.float32)).to(DEV)
    lab = torch.from_numpy(rng.integers(0, 256, n).astype(np.uint8)).to(DEV)
    jit = np.random.default_rng(1).standard_normal((n, 3))
    params = np.array([0.25, 0.75, 3.5, -7.25, 1.0, 12.75, 0.3, 1.1])
    cmax = torch.from_numpy(cv.cpu().numpy().max(0).astype(np.float64)).to(DEV)
    fmm = torch.from_numpy(np.concatenate([f32.cpu().numpy().min(0), f32.cpu().numpy().max(0)]).astype(np.float64)).to(DEV)
    ic = torch.full((n, 4), -7, dtype=torch.int32, device=DEV)
    ifl = torch.full((n, 3), float('nan'), dtype=torch.float32, device=DEV)
    il = torch.full((n,), -7, dtype=torch.int64, device=DEV)
    C.call('osb_aug_input_transforms', C.ptr(cv), 2, C.ptr(f32), 0, C.ptr(lab), None, n, C.ptr(cmax), C.ptr(fmm),
           C.ptr(torch.from_numpy(jit).to(DEV)), params.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 127, 6, None,
           None, C.ptr(ic), C.ptr(ifl), C.ptr(il), C.stream_ptr())
    c_ref = cv.cpu().numpy().copy()
    c_ref[:, :2] = c_ref[:, :2].max(0) - c_ref[:, :2]
    f = f32.cpu().numpy()
    lo, hi = f.min(0), f.max(0)
    f = np.float32(0.25) * f + np.float32(0.75) * ((f - lo) * (255 / (hi - lo)))
    f[:] = np.clip(f + params[2:5], 0, 255)
    f[:] = np.clip(jit * params[5] + f, 0, 255)
    f[:] = A.hsv_shift(f, params[6], params[7])
    assert np.array_equal(ic.cpu().numpy()[:, 0], np.full(n, 6)) and same(ic.cpu().numpy()[:, 1:], c_ref)
    assert same(ifl.cpu().numpy(), (torch.from_numpy(f).float() / 127.5 - 1.).numpy())
    assert same(il.cpu().numpy(), lab.cpu().numpy().astype(np.int64))


def test_a_batch_of_items_feeds_fused_train_step():
    from openscene_b200 import engine, synth, train_mink
    aug = _aug()
    it = aug.DeviceItemAugmenter(voxel_size=0.05, input_color=True)
    seed(3)
    parts = []
    for b in range(8):
        pts = synth.room_points((3.0, 2.5, 1.5), 4, 0.03, seed=b)
        n = len(pts)
        rng = np.random.RandomState(b)
        parts.append(it.point(pts, rng.rand(n, 3) * 255, rng.randint(0, 20, n).astype(np.uint8), batch_index=b))
    coords = torch.cat([p[0] for p in parts])
    feats = torch.cat([p[1] for p in parts])
    labels = torch.cat([p[2] for p in parts])
    assert torch.equal(torch.unique(coords[:, 0]).cpu(), torch.arange(8, dtype=torch.int32))
    model = synth.build_model('MinkUNet18A', 20, seed=0).train().to(DEV)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    loss, pred = train_mink.fused_train_step(eng, opt, coords, feats, labels, ignore_label=255)
    assert torch.isfinite(loss) and pred.shape[0] == coords.shape[0]
