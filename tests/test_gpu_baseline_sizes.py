"""Parity AT BASELINE.json's sizes against the oracle run live (VERDICT r1, 'parity at BASELINE sizes is
self-referential'): the fp32 oracle needs ~2 s for config 1 (MinkUNet18A, ~58k voxels) and ~6 s for config 2
(MinkUNet34C, ~197k voxels) on the GPU box's host cores, so nothing here has to be a self-comparison.

* kernel maps (3^3 at levels 0 and 1, the 2^3 stride-2 map between them): EXACT triple sets (k, c_in, c_out);
* per-point features of the whole network: < 1e-3 relative (north star), against the fp32 oracle;
* a lidar-shaped scene (> 2^9 cells per axis -> the coordinate HASH path at the fine levels, not the occupancy grid);
* the ensemble matcher at Matterport shape (540k voxels, K = 160; run/evaluate.py:302-323).
"""
import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests import match_ref as M
from tests.util import rel_row_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _ckey(c):
    from oracle.me_cpu import _pack
    return _pack(np.asarray(c, dtype=np.int64))


def _sorted_triples(k, kin, kout):
    t = np.stack([k.astype(np.int64), kin, kout], 1)
    return t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]


def _triples_gpu(km, cin, cout):
    nbr = km.nbr.cpu().numpy()
    k, o = np.nonzero(nbr >= 0)
    i = nbr[k, o]
    return _sorted_triples(k, _ckey(cin.cpu().numpy())[i], _ckey(cout.cpu().numpy())[o])


def _triples_oracle(maps, cin, cout):
    ks = np.concatenate([np.full(len(ii), k, dtype=np.int64) for k, (ii, _) in enumerate(maps)])
    ii = np.concatenate([m[0].numpy() for m in maps])
    oo = np.concatenate([m[1].numpy() for m in maps])
    return _sorted_triples(ks, _ckey(cin)[ii], _ckey(cout)[oo])


def _check_maps(cm, om, levels=(1, 2)):
    """3^3 maps at tensor strides `levels`, 2^3 stride-2 maps between consecutive strides: exact."""
    ts = 1
    while ts < max(levels):
        assert cm.stride(ts, 2) == om.stride(ts, 2)
        ts *= 2
    for ts in levels:
        got = cm.sets[ts].coords.cpu().numpy()
        assert len(got) == len(om.coords[ts])
        assert np.array_equal(np.sort(_ckey(got)), np.sort(_ckey(om.coords[ts])))
        km = cm.kernel_map(ts, ts, 3)
        a, b = _triples_gpu(km, cm.sets[ts].coords, cm.sets[ts].coords), _triples_oracle(om.kernel_map(ts, ts, 3), om.coords[ts], om.coords[ts])
        assert a.shape == b.shape and np.array_equal(a, b), f'3^3 map at tensor stride {ts}'
        assert km.num_pairs() == len(b)
    for ts in levels[:-1]:
        km = cm.kernel_map(ts, 2 * ts, 2)
        a = _triples_gpu(km, cm.sets[ts].coords, cm.sets[2 * ts].coords)
        b = _triples_oracle(om.kernel_map(ts, 2 * ts, 2), om.coords[ts], om.coords[2 * ts])
        assert np.array_equal(a, b), f'2^3 stride-2 map {ts}->{2 * ts}'


def _oracle_forward(arch, coords, feats, threads=16):
    from oracle import me_cpu
    torch.set_num_threads(threads)
    model = synth.build_model(arch, 768, seed=0, ME=me_cpu.as_module()).eval()
    sin = me_cpu.SparseTensor(feats, torch.from_numpy(coords))
    with torch.no_grad():
        out = model(sin)
    return out, sin.coordinate_manager


@pytest.mark.parametrize('workload,arch,n_lo,n_hi', [('config1_50k', 'MinkUNet18A', 50_000, 65_000),
                                                      ('config2_200k', 'MinkUNet34C', 190_000, 205_000)])
def test_network_and_maps_against_live_oracle(workload, arch, n_lo, n_hi):
    from openscene_b200 import engine
    c = synth.scene(workload)
    assert n_lo < len(c) < n_hi
    feats = torch.ones(len(c), 3)                                        # dataset/feature_loader.py:184
    ref, om = _oracle_forward(arch, c, feats)
    model = synth.build_model(arch, 768, seed=0).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    out = eng(torch.from_numpy(c).to(DEV), feats.to(DEV))
    err = rel_row_err(out.cpu().numpy(), ref.numpy())
    print(workload, arch, 'engine vs fp32 oracle, per-point rel err', err)
    assert err < 1e-3
    _check_maps(eng.last_cm, om)
    # the module-by-module surface (the unmodified call site run/evaluate.py:289) on the same scene
    import MinkowskiEngine as ME
    with torch.no_grad():
        out_m = model(ME.SparseTensor(feats.to(DEV), torch.from_numpy(c).to(DEV)))
    assert rel_row_err(out_m.cpu().numpy(), ref.numpy()) < 1e-3


def test_lidar_shaped_scene_takes_the_hash_path_and_matches_oracle():
    from openscene_b200 import engine
    c = synth.scene('lidar_80000')
    ext = c[:, 1:].max(0) - c[:, 1:].min(0)
    assert len(c) >= 100_000 and ext[:2].min() > 512                      # too wide for the 2^9 occupancy grid
    feats = torch.ones(len(c), 3)
    ref, om = _oracle_forward('MinkUNet18A', c, feats)
    model = synth.build_model('MinkUNet18A', 768, seed=0).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    out = eng(torch.from_numpy(c).to(DEV), feats.to(DEV))
    cm = eng.last_cm
    assert cm.sets[1].grid is None and cm.sets[2].grid is None            # hash at the fine levels ...
    assert cm.sets[16].grid is not None                                   # ... grid again once the set fits
    err = rel_row_err(out.cpu().numpy(), ref.numpy())
    print('lidar', len(c), 'voxels, per-point rel err', err)
    assert err < 1e-3
    _check_maps(cm, om, levels=(1, 2, 4))


def test_ensemble_matching_at_matterport_shape():
    """run/evaluate.py:302-323 at config 4's shape: N0 = 540k voxels, N_pts = 1.3 N0, K = 160."""
    from openscene_b200 import matching
    from oracle import matching as om
    n_vox = len(synth.scene('config4_matterport'))
    assert 500_000 < n_vox < 580_000
    g = torch.Generator().manual_seed(7)
    f3 = torch.randn(n_vox, 768, generator=g) * (0.2 + torch.rand(n_vox, 1, generator=g))
    f2 = (torch.randn(n_vox, 768, generator=g) * (0.2 + torch.rand(n_vox, 1, generator=g))).half()
    inv = torch.randint(0, n_vox, (int(1.3 * n_vox),), generator=g)
    text = torch.from_numpy(synth.text_embeddings(160))
    s, l, fe, m = matching.match_ensemble(f3.to(DEV), f2.to(DEV), inv.to(DEV), text.to(DEV), return_features=True)
    torch.set_num_threads(16)
    sr, lr, fer, mr = om.match_ensemble(f3, f2, inv, text)
    # against fp64: a choice may differ only where the two maxima's bound intervals overlap (ties between fp16 maxima), the
    # feature is the chosen row bit for bit, every score within its bound, labels by the rule; the oracle obeys the same
    w, n_dis, gap = M.check_ensemble(s, l, fe, m, f3.to(DEV), f2.to(DEV), inv.to(DEV), text.to(DEV), 'tc')
    print('ensemble at Matterport shape: worst', w, 'of the bound;', n_dis, 'choices differ from fp64, largest gap', gap)
    M.check_ensemble(sr.to(DEV), lr.to(DEV), fer.to(DEV), mr.to(DEV), f3.to(DEV), f2.to(DEV), inv.to(DEV), text.to(DEV), 'tc')
