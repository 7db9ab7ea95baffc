"""Torch (CPU) restatement of the FP8 index contract (DESIGN.md, "FP8 index contract"): the e4m3 codes, the per-row
exponents and the dequantized fp16 rows of an FP8 ``SceneIndex``.

Per row: h = the row as fp16 (fp32 is rounded first); a row with a NaN or inf element gets NaN codes (0x7f) and e = 0;
otherwise e is the smallest integer with max|h| <= 448 * 2^e, clamped to [-15, 7], and code = e4m3_rn(clamp(h * 2^-e,
-448, 448)).  d = code * 2^e is exact in fp16.  ``rule`` selects deliberately wrong variants for the negative controls of
the CPU test: 'toward_zero' (truncating rounding), 'exp_plus_one', 'per_tensor' (one exponent for the whole operand),
'flush_subnormals' and 'nan_element' (NaN codes only for the non-finite elements)."""
import torch

E_MIN, E_MAX, F8_MAX = -15, 7, 448.0
NAN_CODE = 0x7f


def _pow2(e):
    """2^e as fp32, exactly, for integer e in [-126, 127]"""
    return ((e.to(torch.int32) + 127) << 23).view(torch.float32)


def _exponent(amax):
    """smallest e in [E_MIN, E_MAX] with amax <= 448 * 2^e (E_MAX when there is none)"""
    e = torch.full(amax.shape, E_MIN, dtype=torch.int32, device=amax.device)
    for k in range(E_MIN, E_MAX):
        e += (amax > F8_MAX * 2.0 ** k).int()
    return e


def _e4m3_toward_zero(x):
    """e4m3 codes of x by truncation: the largest-magnitude code not above |x|"""
    rn = x.to(torch.float8_e4m3fn)
    over = rn.float().abs() > x.abs()
    bits = rn.view(torch.uint8).clone()
    bits[over] -= 1                      # one code toward zero (same sign; 0x00 / 0x80 are never above |x|)
    return bits


def f8_ref(rows, rule=None):
    """rows fp16 / fp32 [n, C] -> (codes uint8 [n, C], exp int8 [n], d fp16 [n, C]), on the rows' device"""
    h = rows.detach().half().float()
    bad = ~torch.isfinite(h).all(1)
    amax = torch.nan_to_num(h.abs(), nan=0.0, posinf=0.0).amax(1)
    if rule == 'per_tensor':
        amax = torch.full_like(amax, float(amax[~bad].max()) if (~bad).any() else 0.0)
    e = _exponent(amax)
    if rule == 'exp_plus_one':
        e = e + 1
    if rule != 'nan_element':
        e[bad] = 0
    x = (h * _pow2(-e)[:, None]).clamp(-F8_MAX, F8_MAX)
    if rule == 'toward_zero':
        codes = _e4m3_toward_zero(torch.nan_to_num(x))
    else:
        codes = torch.nan_to_num(x).to(torch.float8_e4m3fn).view(torch.uint8).clone()
    if rule == 'flush_subnormals':
        sub = (codes & 0x78) == 0
        codes[sub] &= 0x80
    if rule == 'nan_element':
        codes[~torch.isfinite(h)] = NAN_CODE
    else:
        codes[bad] = NAN_CODE
    d = (codes.view(torch.float8_e4m3fn).float() * _pow2(e)[:, None]).half()
    return codes, e.to(torch.int8), d
