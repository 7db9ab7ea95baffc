"""The FP8 index restatement (tests/f8_ref.py) against an independent brute-force rule: for each value the nearest of the
256 e4m3 codes (same sign, ties to the even code), on planted ties, subnormals, saturation, exponent edges and clamps,
zeros, -0 and non-finite rows; and against five mutated rules.  Also the C ABI's refusals of the FP8 entry points, in a
child process (no GPU: they happen before any CUDA call)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.f8_ref import f8_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _e4m3_table():
    """float64 value of every code (NaN for 0x7f / 0xff), from the format's definition"""
    v = np.empty(256)
    for c in range(256):
        s, ex, m = c >> 7, (c >> 3) & 15, c & 7
        if ex == 15 and m == 7:
            v[c] = np.nan
        elif ex == 0:
            v[c] = (m / 8) * 2.0 ** -6
        else:
            v[c] = (1 + m / 8) * 2.0 ** (ex - 7)
        v[c] = -v[c] if s else v[c]
    return v


TABLE = _e4m3_table()


def brute(rows):
    """(codes uint8 [n, C], exp int8 [n], d float64 [n, C]) by exhaustive search, in float64"""
    h = rows.detach().cpu().half().double().numpy()
    n, c = h.shape
    codes = np.full((n, c), 0x7f, np.uint8)
    exps = np.zeros(n, np.int8)
    signed = np.signbit(TABLE)
    finite = ~np.isnan(TABLE)
    for i in range(n):
        if not np.isfinite(h[i]).all():
            continue
        amax = np.abs(h[i]).max()
        e = next((k for k in range(-15, 8) if amax <= 448.0 * 2.0 ** k), 7)
        exps[i] = e
        x = np.clip(h[i] * 2.0 ** -e, -448.0, 448.0)
        dist = np.abs(x[:, None] - TABLE[None, :])
        dist[:, ~finite] = np.inf
        dist[np.signbit(x)[:, None] != signed[None, :]] = np.inf      # the code keeps the sign, -0 included
        best = dist.min(1, keepdims=True)
        cand = dist == best
        even = cand & ((np.arange(256) & 1) == 0)[None, :]
        pick = np.where(even.any(1), even.argmax(1), cand.argmax(1))
        assert (cand.sum(1) <= 2).all()
        codes[i] = pick
    d = TABLE[codes] * (2.0 ** exps.astype(np.float64))[:, None]
    return codes, exps, d


def _planted(c=16):
    """rows of width c, each testing one edge of the rule; unused slots are zero"""
    rows = []

    def row(*vals):
        r = torch.zeros(c, dtype=torch.float64)
        r[:len(vals)] = torch.tensor(vals, dtype=torch.float64)
        rows.append(r)
    # e = 0 (amax 448): ties between neighbouring codes at several binades, to the even code
    row(448, 1.0625, 1.1875, 1.3125, 17, 19, 25, 27, 2.0 ** -7 * 1.0625, 240 + 8, 224 + 8, -1.0625, -1.1875, 0.5 + 1 / 32)
    # e = 0: subnormals of e4m3 (|x| < 2^-6), their ties (to 0 and to the even code) and the smallest subnormal
    row(448, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 5 * 2.0 ** -10, 7 * 2.0 ** -10, 2.0 ** -6 - 2.0 ** -10, 2.0 ** -11,
        -(2.0 ** -10), -3 * 2.0 ** -10, 15 * 2.0 ** -10, 2.0 ** -12, 6 * 2.0 ** -9, 13 * 2.0 ** -10)
    # 464 / 480: e = 1 (a tie between 224 and 240 at the top binade, and 240 exactly)
    row(464, 480, -464, 463, 450)
    # saturation: amax above 448 * 2^7 clamps e to 7, and the codes to +-448
    row(65504, 59392, 61440, 57344, -65504, -57344, 57376, 1.0, -0.0)
    # amax exactly 448 * 2^e, and one fp16 ulp above it
    row(56, 1, 3)
    row(56.03125, 1, 3)
    row(-448 * 2.0 ** -10, 2.0 ** -20)
    row(448 * 2.0 ** -10 + 2.0 ** -12, 2.0 ** -20)
    # the lower clamp: amax far below 448 * 2^-15 (fp16 subnormals), e = -15
    row(2.0 ** -24, 3 * 2.0 ** -24, 2.0 ** -20, -(2.0 ** -14), 2.0 ** -16 * 5)
    row(448 * 2.0 ** -15, 2.0 ** -24, 2.0 ** -23)
    # zero rows, -0 kept, and a row of only -0
    row()
    row(-0.0, 0.0, -0.0, 2.0 ** -10)
    rows.append(torch.full((c,), -0.0, dtype=torch.float64))
    # non-finite rows: NaN, +inf, -inf among finite values
    row(1, float('nan'), 2)
    row(float('inf'), 1)
    row(3, float('-inf'), -0.0)
    return torch.stack(rows)


def _check(rows):
    codes, e, d = f8_ref(rows)
    bc, be, bd = brute(rows)
    assert np.array_equal(codes.numpy(), bc)
    assert np.array_equal(e.numpy(), be)
    assert d.dtype == torch.float16
    dd = d.double().numpy()
    fin = ~np.isnan(bd)
    assert np.array_equal(np.isnan(dd), ~fin)
    assert np.array_equal(dd[fin], bd[fin])                          # d = code * 2^e exactly, in float64
    assert np.array_equal(np.signbit(dd[fin]), np.signbit(bd[fin]))
    return codes, e, d


def test_planted_rows_against_the_brute_force_rule():
    rows = _planted()
    same = lambda t: torch.nan_to_num(t, nan=7.0)                                        # noqa: E731
    assert torch.equal(same(rows.half().double()), same(rows))         # every planted value is an fp16 number
    codes, e, d = _check(rows)
    assert e.tolist() == [0, 0, 1, 7, -3, -2, -10, -9, -15, -15, -15, -15, -15, 0, 0, 0]
    assert codes[0, 1] == 0x38 and codes[0, 2] == 0x3a               # 1.0625 -> 1, 1.1875 -> 1.25
    assert codes[1, 2] == 0x00 and codes[1, 3] == 0x02                # 2^-10 -> +0, 3 * 2^-10 -> 2 * 2^-9
    assert codes[1, 1] == 0x01 and d[1, 1].item() == 2.0 ** -9
    assert codes[2, 0] == 0x76 and codes[2, 1] == 0x77                 # 232 -> 224 (even), 240
    assert (codes[3, :3] == 0x7e).all() and codes[3, 4] == 0xfe       # saturated to +-448, d = +-57344
    assert d[3, 0].item() == 57344.0
    assert codes[8, 0] == 0x01 and d[8, 0].item() == 2.0 ** -24        # the smallest fp16 subnormal
    assert codes[11, 0] == 0x80 and codes[11, 1] == 0x00              # -0 keeps its sign
    assert (codes[10] == 0).all() and (codes[12] == 0x80).all() and (codes[13:] == 0x7f).all()
    assert torch.isnan(d[13:]).all()


@pytest.mark.parametrize('scale', [1e-6, 1e-3, 0.05, 1.0, 300.0, 4e4])
def test_random_rows_against_the_brute_force_rule(scale):
    g = torch.Generator().manual_seed(int(scale * 1000) + 1)
    rows = torch.randn(24, 64, generator=g, dtype=torch.float64) * scale
    rows[::5] *= torch.rand(rows[::5].shape, generator=g, dtype=torch.float64) ** 6        # wide dynamic range
    _check(rows.half())


def test_fp32_input_is_its_half():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(40, 512, generator=g) * 0.05
    x[3, 7] = 7e4                                                     # rounds to inf in fp16: a non-finite row
    x[4] = torch.randn(512, generator=g) * 1e-6
    x[5, :4] = torch.tensor([1.0 + 2 ** -12, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, 2 ** -25])
    a, b = f8_ref(x), f8_ref(x.half())
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int16) if u.dtype == torch.float16 else u,
                           v.view(torch.int16) if v.dtype == torch.float16 else v)
    assert (a[0][3] == 0x7f).all() and int(a[1][3]) == 0
    _check(x)


@pytest.mark.parametrize('rule', ['toward_zero', 'exp_plus_one', 'per_tensor', 'flush_subnormals', 'nan_element'])
def test_mutated_rules_fail(rule):
    rows = _planted()
    bc, be, _ = brute(rows)
    codes, e, _ = f8_ref(rows, rule=rule)
    assert not (np.array_equal(codes.numpy(), bc) and np.array_equal(e.numpy(), be)), rule


def test_bad_storage_is_refused():
    from openscene_b200.search import SceneIndex
    for bad in ('bf16', 'e4m3', None, 8):
        with pytest.raises(ValueError, match='storage'):
            SceneIndex(100, 768, device='cuda', storage=bad)


_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
out = {}
A = 1 << 20            # a 16-byte aligned non-NULL placeholder: never dereferenced, every call is refused first
def off(*v):
    return (C.I64 * len(v))(*v)
def q(tag, rows=A, c=768, n=10, codes=A, exp=A):
    out[tag] = [L.osb_index_quantize_f8(rows, 1, n, c, codes, exp, None), (L.osb_last_error() or b'').decode()]
q('q_width', c=640); q('q_n0', n=0); q('q_null_rows', rows=None); q('q_null_codes', codes=None); q('q_null_exp', exp=None)
q('q_misaligned', rows=A + 2); q('q_misaligned_codes', codes=A + 8)
def s(tag, codes=A, exp=A, c=768, k=2):
    r = L.osb_search_f8(codes, exp, A, 10, c, off(0, 10), A, 1, A, 4, k, None, A, A, A, A, A, None, A, 1 << 30, None)
    out[tag] = [r, (L.osb_last_error() or b'').decode()]
s('s_null_exp', exp=None); s('s_width', c=640); s('s_misaligned', codes=A + 4); s('s_k', k=33)
def h(tag, codes=A, exp=A, c=768):
    r = L.osb_search_hits_f8(codes, exp, A, 10, c, off(0, 10), 1, A, 4, A, A, 5, A, A, A, A, 1 << 30, None)
    out[tag] = [r, (L.osb_last_error() or b'').decode()]
h('h_null_exp', exp=None); h('h_width', c=1024); h('h_misaligned', codes=A + 8)
print('RESULT ' + json.dumps(out))
'''


def test_f8_refusals_happen_on_the_host_with_a_message():
    p = subprocess.run([sys.executable, '-c', _CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
    expect = {'q_width': 'width', 'q_n0': 'N=', 'q_null_rows': 'NULL', 'q_null_codes': 'NULL', 'q_null_exp': 'NULL',
              'q_misaligned': 'aligned', 'q_misaligned_codes': 'aligned', 's_null_exp': 'exponents',
              's_width': 'width', 's_misaligned': 'aligned', 's_k': 'k=', 'h_null_exp': 'exponents', 'h_width': 'width',
              'h_misaligned': 'aligned'}
    assert sorted(res) == sorted(expect)
    for tag, (rc, err) in res.items():
        assert rc != 0, f"{tag}: accepted"
        assert expect[tag] in err, f"{tag}: {err!r}"
        assert err.startswith('osb_index_quantize_f8' if tag[0] == 'q' else 'osb_search_f8' if tag[0] == 's'
                              else 'osb_search_hits_f8'), err
