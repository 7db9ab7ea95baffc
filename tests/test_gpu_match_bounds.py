"""Every score of the matching kernels within its fp64 bound (tests/match_ref.py, DESIGN.md section 2), and every label and
row maximum consistent with the kernel's own scores.

Tensor-core route (k_match_tc) in this process, CUDA-core route (k_match_scores, k_match_ensemble; OSB_MATCH_SIMT=1, read
once per process) in a child.  Cases: K at both sides of every 96-row pass edge from one to five passes, C = 512 / 768, fp32
and fp16 sources with and without normalisation, n_pts around the 128-point tile and above the CUDA-core grid cap of 8448
warps, inds_reverse absent / shorter / longer than n_vox / heavily repeated.  The ensemble branch: a point's 3-D / 2-D choice
may differ from the fp64 decision only where the bound intervals of the two normalised maxima overlap, the ensemble feature is
bit for bit the source row the kernel's own choice picked, and the final scores are within the bound of that feature.  The
folded head (osb_folded_head_finish) on fp32 z with several columns per lane."""
import os
import subprocess
import sys

import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import matching, synth
from tests import match_ref as M

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KS = [1, 2, 95, 96, 97, 191, 192, 193, 383, 384, 385, 479, 480]
NPTS = [1, 127, 128, 129, 20000]
MODES = ['none', 'short', 'long', 'repeat']


def point_indices(n_pts, mode, g):
    """(n_vox, inds_reverse or None): absent, a subset of a larger voxel set, longer than the voxel set, few voxels repeated"""
    if mode == 'none':
        return n_pts, None
    if mode == 'short':
        n_vox = n_pts + 53
        return n_vox, torch.randperm(n_vox, generator=g)[:n_pts].to(DEV)
    if mode == 'long':
        n_vox = max(1, n_pts // 3)
        return n_vox, torch.randint(0, n_vox, (n_pts,), generator=g).to(DEV)
    n_vox = n_pts + 7
    return n_vox, torch.randint(0, min(3, n_vox), (n_pts,), generator=g).to(DEV)


def cases(k):
    """(c, n_pts, mode) per K: every width, and across the K list every n_pts / mode pairing"""
    i = KS.index(k)
    out = [(c, NPTS[(2 * i + j) % 5], MODES[(i + j) % 4]) for j, c in enumerate((512, 768))]
    if k in (1, 97, 480):
        out.append((768, 20000, MODES[i % 4]))
    return out


def _feats(n, c, g):
    f = torch.randn(n, c, generator=g) * (0.2 + torch.rand(n, 1, generator=g))
    return f.to(DEV)


def check_products(k, route):
    """the four products of one K on every case; returns {product: worst fraction of the bound}"""
    worst = {}
    for c, n_pts, mode in cases(k):
        g = torch.Generator().manual_seed(1000 * k + c + n_pts)
        t = torch.from_numpy(synth.text_embeddings(k, c, seed=k)).to(DEV)
        n_vox, inv = point_indices(n_pts, mode, g)
        x = _feats(n_vox, c, g)
        for f16 in (False, True):
            xf = x.half() if f16 else x
            for normalize in (False, True):
                s, lab, smax = matching._scores(xf, inv, t, normalize, want_smax=True)
                r = M.check_scores(s, xf, inv, t, normalize, route)
                M.check_labels(s, lab, smax)
                key = ('normalised' if normalize else 'plain') + (' fp16' if f16 else ' fp32')
                worst[key] = max(worst.get(key, 0.0), r)
    return worst


def check_ensemble(k, route):
    """returns (worst fraction of the final scores' bound, disagreeing points, largest fp64 gap among them)"""
    worst, n_dis, gap = 0.0, 0, 0.0
    for c, n_pts, mode in cases(k):
        g = torch.Generator().manual_seed(7 * k + c + n_pts)
        t = torch.from_numpy(synth.text_embeddings(k, c, seed=k + 1)).to(DEV)
        n_vox, inv = point_indices(n_pts, mode, g)
        f3, f2 = _feats(n_vox, c, g), _feats(n_vox, c, g).half()
        s, lab, fe, m = matching.match_ensemble(f3, f2, inv, t, return_features=True)
        w, nd, gp = M.check_ensemble(s, lab, fe, m, f3, f2, inv, t, route)
        worst, n_dis, gap = max(worst, w), n_dis + nd, max(gap, gp)
    return worst, n_dis, gap


def run_all(route, ks=KS):
    out = {}
    for k in ks:
        for key, r in check_products(k, route).items():
            out[key] = max(out.get(key, 0.0), r)
        w, n_dis, gap = check_ensemble(k, route)
        out['ensemble'] = max(out.get('ensemble', 0.0), w)
        out['mask disagreements'] = out.get('mask disagreements', 0) + n_dis
        out['largest disagreeing gap'] = max(out.get('largest disagreeing gap', 0.0), gap)
    print(f'BOUNDS {route}: ' + ', '.join(f'{k} {v:.4g}' for k, v in out.items()), flush=True)
    return out


@pytest.mark.parametrize('k', KS)
def test_tensor_core_route_within_bounds(k):
    run_all('tc', [k])


_SIMT_CHILD = r'''
import sys
sys.path.insert(0, sys.argv[1])
from tests.test_gpu_match_bounds import run_all
run_all('simt')
print('SIMT_OK')
'''


def test_cuda_core_route_within_bounds():
    p = subprocess.run([sys.executable, '-c', _SIMT_CHILD, ROOT], capture_output=True, text=True, timeout=1200,
                       env=dict(os.environ, OSB_MATCH_SIMT='1'))
    print(p.stdout[-3000:])
    assert p.returncode == 0 and 'SIMT_OK' in p.stdout, p.stdout[-2000:] + p.stderr[-3000:]


# ------------------------------------------------------------------------------------------------ folded head
def folded_finish(z, c_norm, k):
    n, ld = z.shape
    scores = torch.empty((n, k), dtype=torch.float16, device=DEV)
    label = torch.empty(n, dtype=torch.int64, device=DEV)
    smax = torch.empty(n, dtype=torch.float32, device=DEV)
    C.call('osb_folded_head_finish', C.ptr(z), n, ld, c_norm, k, C.ptr(scores), C.ptr(label), C.ptr(smax), C.stream_ptr())
    return scores, label, smax


@pytest.mark.parametrize('k', [1, 20, 33, 160, 480])
def test_folded_head_finish_within_bounds(k):
    """score = fp16(z_k / (|z_L| + 1e-5)): one lane sums c_norm / 32 squares by FMA and 5 shuffle adds, then sqrt, +1e-5 and
    the division each round once in fp32, so the value before the fp16 rounding is within (depth / 2 + 3) 2^-24 of the
    fp64 quotient"""
    c_norm, n = 96, 20000
    ld = c_norm + k + 13
    g = torch.Generator().manual_seed(k)
    z = (torch.randn(n, ld, generator=g) * torch.exp2(torch.randint(-6, 7, (n, 1), generator=g).float())).to(DEV)
    s, lab, smax = folded_finish(z, c_norm, k)
    zd = z.double()
    S = zd[:, c_norm:c_norm + k] / (zd[:, :c_norm].norm(dim=1, keepdim=True) + 1e-5)
    rel = ((-(-c_norm // 32) + 5) / 2 + 3) * M.U32 * (1 + 2.0 ** -10)
    B = rel * S.abs() + 0.5 * M.ulp16(S.abs() * (1 + rel))
    r = M.score_ratio(s, S, B)
    print(f'BOUNDS folded head k={k}: {r:.4g}')
    assert r <= 1.0
    M.check_labels(s, lab, smax)
