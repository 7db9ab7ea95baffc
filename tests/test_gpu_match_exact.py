"""Bit-exact probes of the matching kernels, and one label rule for the non-vote kernels.

Operands lie on a dyadic grid (tests/match_ref.py: dyadic_text, dyadic_points) small enough that every partial sum an fp32
accumulator can form is an exact multiple of the grid below 2^24 grid units, so every route must return fp16_rn(exact sum)
bit for bit: k_match_tc, k_match_scores (OSB_MATCH_SIMT=1, in a child), the vote epilogue k_match_tc_vote with the paired and
the two-access store (and the CUDA-core vote route in the child), and k_match_ensemble with its tensor-core counterpart,
whose ensemble feature must also be the chosen source row bit for bit.  fp16 rows normalised in the kernel have a power-of-
two norm (down to 2^-5, where fp16(norm + 1e-5) still equals the norm), so d is exact and x rcp(d) = x / d.  fp32 sources
carry a perturbation below half an fp16 ulp that the kernel's rounding must remove.  Planted rows: exact ties between the
text rows 95/96, 191/192, 383/384, 0/K-1 and between interleaved column pairs of one lane group (the lower column wins);
finite sums that overflow fp16 to +inf at two tied columns, rows whose every score overflows to -inf; scores that cancel to
zero; an all-zero row (normalised: divided by fp16(1e-5)).  An exact zero may come back as either sign.

Label rule (match.cu, DESIGN.md section 2): on rows with NaN scores, rows of only -inf and rows of only NaN, fed through the
feature (or through z for the folded head), every non-vote kernel takes the lowest column holding the largest non-NaN score,
0 when there is none, and they agree with each other."""
import math
import os
import subprocess
import sys

import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import matching
from tests import match_ref as M
from tests.test_gpu_match_bounds import KS, NPTS, MODES, ROOT, folded_finish, point_indices

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
KINDS = ['f32', 'f16', 'f16norm']
TIE_PAIRS = [(95, 96), (191, 192), (383, 384), (2, 8), (1, 6), (3, 4), (0, None)]


def tie_pairs(k):
    used, out = set(), []
    for j1, j2 in TIE_PAIRS:
        j2 = k - 1 if j2 is None else j2
        if j2 < k and j1 != j2 and j1 not in used and j2 not in used:
            used |= {j1, j2}
            out.append((j1, j2))
    return out


def probe(k, c, n_pts, mode, kind, g):
    """(features as the kernel reads them, exact fp64 operand rows, inds_reverse, text, planted row count)"""
    t = M.dyadic_text(k, c, g)
    pairs = tie_pairs(k)
    for j1, j2 in pairs:
        t[j2] = t[j1]
    td = t.double()
    norm = kind == 'f16norm'
    planted = [td[j1] * 2.0 for j1, _ in pairs]                            # norm 2: a tie at the row maximum
    zero = torch.zeros(c, dtype=torch.float64)
    planted.append(zero)
    cancel = zero.clone()
    cancel[:8], cancel[8:16] = 0.5, -0.5                                     # every score exactly 0 (norm 2)
    planted.append(cancel)
    if not norm:
        mixed = cancel.clone()
        mixed[16:] = -td[:, 16:].sum(0).sign() * (td[:, 16:] != 0).any(0) * 0.25
        planted.append(mixed)                                                # some scores 0, others of both signs
        if pairs:
            planted.append(td[pairs[0][0]] * 2.0 ** 16)                      # 65536 at a tied pair: +inf, +inf
        allneg = zero.clone()
        allneg[:16] = -M.FP16_MAX_FINITE                                     # every score -131008: -inf
        planted.append(allneg)
    n_vox, inv = point_indices(n_pts, mode, g)
    x = M.dyadic_points(n_vox, c, g, norm_pow2=norm)
    n_pl = min(n_vox, len(planted))
    x[:n_pl] = torch.stack(planted[:n_pl])
    if inv is not None:
        m = min(n_pts, n_pl)
        inv[:m] = torch.arange(m, device=DEV)
    a = x / x.norm(dim=1, keepdim=True).clamp(min=1e-300) if norm else x
    if kind == 'f32':
        noise = 0.2 * M.ulp16(x) * torch.where(torch.rand(x.shape, generator=g) < 0.5, -1.0, 1.0).double()
        feat = (x + noise * (x != 0)).float()
        assert torch.equal(feat.half().double(), x)
    else:
        feat = x.half()
    return feat.to(DEV), a.to(DEV), inv, t.to(DEV), n_pl


def same_or_zero(s, ref):
    """bit-identical, except that an exact zero may carry either sign"""
    return bool(((s.view(torch.int16) == ref.view(torch.int16)) | ((s == 0) & (ref == 0))).all())


def expect(a, inv, t):
    ai = a[inv] if inv is not None else a
    bits = M.exact_budget_bits(ai, t)
    assert bits < 24, ('budget', bits)
    return M.fp16_rn(ai @ t.double().t()), bits


def vote(feat, inv, t, normalize, store):
    n_pts = inv.shape[0] if inv is not None else feat.shape[0]
    k = t.shape[0]
    s = torch.empty((n_pts, k), dtype=torch.float16, device=DEV)
    lc = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    la = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    C.call('osb_match_vote', C.ptr(feat), int(feat.dtype == torch.float16), feat.shape[0], feat.shape[1], C.ptr(inv), n_pts,
           C.ptr(t), k, int(normalize), C.ptr(s), C.ptr(store), C.ptr(lc), C.ptr(la), C.stream_ptr())
    return s, lc, la


def ensemble(f3, f2, inv, sel3, sel2, t):
    n_pts = inv.shape[0] if inv is not None else f3.shape[0]
    k, c = t.shape
    s = torch.empty((n_pts, k), dtype=torch.float16, device=DEV)
    lab = torch.empty(n_pts, dtype=torch.int64, device=DEV)
    fe = torch.empty((n_pts, c), dtype=torch.float16, device=DEV)
    C.call('osb_match_ensemble', C.ptr(f3), C.ptr(f2), f3.shape[0], c, C.ptr(inv), n_pts, C.ptr(sel3), C.ptr(sel2), C.ptr(t), k,
           C.ptr(s), C.ptr(lab), C.ptr(fe), C.stream_ptr())
    return s, lab, fe


def run_probes(k, route):
    """every case of one K on the current route; returns the largest budget (log2 of 2^24's share)"""
    worst = 0.0
    i = KS.index(k)
    for j, (c, kind) in enumerate([(c, kd) for c in (512, 768) for kd in KINDS]):
        n_pts, mode = NPTS[(i + j) % 5], MODES[(i + 2 * j) % 4]
        if k in (2, 96, 480) and j == 0:
            n_pts = 20000
        g = torch.Generator().manual_seed(31 * k + 7 * j)
        feat, a, inv, t, n_pl = probe(k, c, n_pts, mode, kind, g)
        norm = kind == 'f16norm'
        ref, bits = expect(a, inv, t)
        worst = max(worst, bits)
        tag = (route, k, c, kind, n_pts, mode)
        s, lab, smax = matching._scores(feat, inv, t, norm, want_smax=True)
        assert same_or_zero(s, ref), ('scores', tag, int((s.view(torch.int16) != ref.view(torch.int16)).sum()))
        M.check_labels(ref, lab, smax)
        m = min(n_pts, n_pl, len(tie_pairs(k)))                               # planted tie rows come first
        assert lab[:m].tolist() == [p[0] for p in tie_pairs(k)][:m], ('tie', tag, lab[:m].tolist())
        # the vote: paired 4-byte store (K even, aligned) and the two-access store (offset by one element)
        n = ref.shape[0]
        for offset in (0, 1):
            flat = torch.zeros(n * k + 1, dtype=torch.float16, device=DEV)
            store = flat[offset:offset + n * k].view(n, k)
            sv, lc, la = vote(feat, inv, t, norm, store)
            assert same_or_zero(sv, ref) and same_or_zero(store, ref), ('vote', offset, tag)
            first = ref.float().cpu().max(1)[1].to(DEV)                      # no NaN here: torch's CPU rule = first max
            assert torch.equal(lc, first) and torch.equal(la, first), ('vote labels', offset, tag)
        if kind == 'f32':
            f2 = M.dyadic_points(feat.shape[0], c, g).half().to(DEV)
            sel3 = torch.randint(0, 3, (n,), generator=g).float().to(DEV)
            sel2 = torch.randint(0, 3, (n,), generator=g).float().to(DEV)    # ties keep the 3-D feature (strict <)
            se, le, fe = ensemble(feat, f2, inv, sel3, sel2, t)
            x3, x2 = (feat[inv], f2[inv]) if inv is not None else (feat, f2)
            chosen = torch.where((sel3 < sel2)[:, None], x2, x3.half())
            assert torch.equal(fe.view(torch.int16), chosen.view(torch.int16)), ('ensemble feature', tag)
            eref, _ = expect(chosen.double(), None, t)
            assert same_or_zero(se, eref), ('ensemble scores', tag)
            M.check_labels(eref, le)
    return worst


def nan_rows(c, k):
    """fp32 rows: +inf on a column where some text rows are 0 (NaN there, +-inf elsewhere), NaN, every score -inf, finite"""
    g = torch.Generator().manual_seed(k + c)
    t = M.dyadic_text(k, c, g).to(DEV)
    td = t.double()
    both = ((td[:, 16:] == 0).any(0) & (td[:, 16:] != 0).any(0)).nonzero()
    col = int(both[0]) + 16 if len(both) else 16
    x = M.dyadic_points(4, c, g).float()
    x[0, col] = math.inf
    x[1, 5] = math.nan
    x[2, :16] = -1e6                                                         # fp16 -inf on the shared positive columns
    return x.to(DEV), t


def label_rule_labels():
    """labels of every non-vote kernel on the NaN / -inf rows of the current route"""
    out = {}
    for k in (1, 2, 40, 97):
        for c in (512, 768):
            x, t = nan_rows(c, k)
            s, lab, smax = matching._scores(x, None, t, False, want_smax=True)
            M.check_labels(s, lab, smax)
            assert lab[1:3].tolist() == [0, 0]
            assert bool(torch.isnan(s[1].float()).all()) and bool((s[2].float() == -math.inf).all())
            out[('scores', k, c)] = lab.tolist()
            z = torch.zeros(4, dtype=torch.float32, device=DEV)
            for sel3, sel2, f2 in ((z, z, x.half()), (z, z + 1, x.half())):          # the 3-D row, then the 2-D row
                se, le, _ = ensemble(x, f2, None, sel3, sel2, t)
                M.check_labels(se, le)
                out[('ensemble', k, c, float(sel2[0]))] = le.tolist()
            assert len({tuple(v) for kk, v in out.items() if kk[1:3] == (k, c)}) == 1, out
    # the folded head on z: the same rule with several columns per lane (K = 40)
    k, c_norm = 40, 96
    z = torch.randn(4, c_norm + k + 8, generator=torch.Generator().manual_seed(3)).to(DEV)
    sc = z[:, c_norm:c_norm + k]
    sc[0, :] = -1.0
    sc[0, [0, 2, 33]] = math.nan
    sc[0, [35, 37]] = 3.0                                                    # the first maximum, behind NaNs in lanes 0 / 2
    z[1, 7] = math.nan                                                       # NaN norm: every score NaN
    sc[2, :] = -math.inf
    s, lab, smax = folded_finish(z, c_norm, k)
    M.check_labels(s, lab, smax)
    assert lab[:3].tolist() == [35, 0, 0], lab.tolist()
    out['folded'] = lab.tolist()
    return out


def _check_all(route):
    bits = max(run_probes(k, route) for k in KS)
    lab = label_rule_labels()
    print(f'EXACT {route}: every probe bit-identical, largest budget 2^{bits:.2f} of 2^24', flush=True)
    return lab


@pytest.mark.parametrize('k', KS)
def test_tensor_core_probes_are_bit_exact(k):
    print(f'EXACT tc k={k}: largest budget 2^{run_probes(k, "tc"):.2f} of 2^24')


def test_label_rule_on_nan_and_inf_rows():
    label_rule_labels()


_SIMT_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from tests.test_gpu_match_exact import _check_all
lab = _check_all('simt')
print('LABELS ' + json.dumps({repr(k): v for k, v in lab.items()}))
print('SIMT_OK')
'''


def test_cuda_core_probes_and_label_rule_agree_with_tensor_cores():
    p = subprocess.run([sys.executable, '-c', _SIMT_CHILD, ROOT], capture_output=True, text=True, timeout=1200,
                       env=dict(os.environ, OSB_MATCH_SIMT='1'))
    print(p.stdout[-3000:])
    assert p.returncode == 0 and 'SIMT_OK' in p.stdout, p.stdout[-2000:] + p.stderr[-3000:]
    import json
    simt = json.loads([l for l in p.stdout.splitlines() if l.startswith('LABELS ')][-1][len('LABELS '):])
    tc = {repr(k): v for k, v in label_rule_labels().items()}
    assert simt == tc
