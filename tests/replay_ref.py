"""fp64 references and error bounds for the convolution entry points of libosb200, shared by
tests/test_gpu_launch_replay.py (every launch of the engine replayed on its own operands), tests/test_gpu_conv_exact.py
(bit-exact probes of the tensor-core arithmetic), tests/test_gpu_conv_f32.py and tests/test_gpu_me_module_exact.py (the
CUDA-core kernels and the module surface) and their CPU self-checks tests/test_replay_ref_cpu.py and
tests/test_f32conv_ref_cpu.py.  Every function runs on CPU or CUDA tensors.

Bounds (DESIGN.md section 2): a tensor-core result y and its fp64 reference y^ computed from the operands the launch read
satisfy, element by element,
    |y - y^| <= c * 2^-16 * A      (+ 2^-17 |y^| when y is written as split rows)
with A = sum |x| |W| (wgrad: sum |x| |g|), scaled through the epilogue (|scale| A + |shift| + |res|), and c from the
accumulation depth of the kernel (``c_forward``, ``c_wgrad``, ``c_fma``)."""
import math

import torch

# one tensor-core accumulation step (a K16 slice of wgmma added to the fp32 accumulator, or one fp32 add of a reduction):
# the 16 products and the accumulator are aligned to the largest exponent and truncated, each losing less than one unit of
# 2^-23 of the largest, and the sum is normalised once more (Fasi, Higham, Mikaitis, Pranesh, "Numerical behavior of NVIDIA
# tensor cores", PeerJ CS 2021): at most 18 x 2^-23 of the magnitudes the step adds
STEP = 18 * 2.0 ** -23
# weight split residual |W - Whi - Wlo| <= 2^-18 |W| and the omitted lo*Wlo <= 2^-18 |x||W| (with the 1 + 2^-8 of |hi| <= |x|)
SPLIT_C = 2.0 ** 16 * 2.0 ** -17 * (1 + 2.0 ** -7)
OUT_SPLIT = 2.0 ** -17


def c_forward(K, cin):
    """osb_conv_fwd_tc / chain / dense transposed: 3 products x K offsets x cin/16 K16 steps, one split-K partial per
    (offset, 32-channel block) at most, 3 epilogue roundings."""
    steps = 3 * K * -(-cin // 16) + K * -(-cin // 32) + 3
    return SPLIT_C + 2.0 ** 16 * steps * STEP


def wgrad_plan(n_out, K, cin, cout):
    """(n_rs, rows_per_rs) of osb_conv_wgrad_tc (csrc/conv_wgrad_tc.cu wgrad_plan)"""
    n_mt, n_nt = (cin // 32 + 1) // 2, (cout // 32 + 3) // 4
    base = K * n_mt * n_nt
    chunks = -(-n_out // 128)
    rs = max(1, -(-264 // base))
    rs = min(rs, max(1, chunks // 4))
    rows_per_rs = -(-chunks // rs) * 128
    return -(-n_out // rows_per_rs), rows_per_rs


def c_wgrad(n_out, K, cin, cout):
    """all four quadrants are exact products: only the accumulation over a row range (K16 steps), the quadrant and row-range
    reduce count"""
    n_rs, rpr = wgrad_plan(n_out, K, cin, cout)
    return 2.0 ** 16 * (rpr // 16 + 4 * n_rs + 4) * STEP


def c_fma(n_terms):
    """fp32 FMA chains on CUDA cores (stem, osb_conv_fwd_f32): fp32 operands, one rounding of 2^-24 per term and epilogue"""
    return 2.0 ** 16 * (n_terms + 3) * 2.0 ** -24


# ------------------------------------------------------------------ CUDA-core fp32 kernels (csrc/conv_f32.cu)
# Every output element of the CUDA-core kernels is an fp32 FMA chain, possibly followed by float atomic adds of per-block
# partials in any order.  To first order each rounding costs 2^-24 of the magnitudes it has summed, so with `depth` the
# longest chain of roundings any one term passes through, |y - y^| <= (depth + 3) 2^-24 A (c_fma(depth) in units of
# 2^-16 A), valid while depth 2^-24 << 1.
THIN_COUT, THIN_SMEM_MAX = 32, 96 * 1024              # k_conv_fwd_thin: lane = output channel, weights in shared memory
WG_ROWS = 4096                                         # k_conv_wgrad_f32: rows per block (one atomic partial each)
THIN_WG_ROWS, THIN_WG_GRID, THIN_WG_KMAX = 128, 132 * 4, 8 * 16    # k_conv_wgrad_thin: chunk rows, grid cap, offsets


def f32_dispatch(entry, cin, cout, K, has_nbr, ld_in=None, transpose_w=False):
    """which kernel osb_conv_fwd_f32 ('fwd') / osb_conv_wgrad_f32 ('wgrad') launches for these arguments:
    'fwd_thin', 'fwd_generic', 'wgrad_thin' or 'wgrad_generic' (a restatement of the host code's dispatch)"""
    if entry == 'fwd':
        ld_in = cin if ld_in is None else ld_in
        thin = (has_nbr and not transpose_w and cout == THIN_COUT and 1 <= cin <= 4 and ld_in == cin
                and K * cin * THIN_COUT * 4 <= THIN_SMEM_MAX)
        return 'fwd_thin' if thin else 'fwd_generic'
    assert entry == 'wgrad'
    thin = has_nbr and cout == THIN_COUT and cin <= 4 and K <= THIN_WG_KMAX
    return 'wgrad_thin' if thin else 'wgrad_generic'


def f32_fwd_depth(K, cin):
    """both forwards: one thread owns an output element and runs K cin FMAs in one chain (absent neighbours and padded
    channels add exact zeros)"""
    return K * cin


def thin_wgrad_grid(n_out):
    return min(-(-n_out // THIN_WG_ROWS), THIN_WG_GRID)


def f32_wgrad_depth(kernel, n_out):
    """generic: at most WG_ROWS FMAs in a block's row chunk, then ceil(n_out / WG_ROWS) atomic adds in any order;
    thin: a block walks ceil(n_chunks / grid) chunks of THIN_WG_ROWS rows in one register, then one atomic add per block"""
    if kernel == 'wgrad_generic':
        return min(n_out, WG_ROWS) + -(-n_out // WG_ROWS)
    assert kernel == 'wgrad_thin'
    n_chunks = -(-n_out // THIN_WG_ROWS)
    grid = thin_wgrad_grid(n_out)
    return -(-n_chunks // grid) * THIN_WG_ROWS + grid


def f32_depth(kernel, K, cin, n_out):
    return f32_fwd_depth(K, cin) if kernel.startswith('fwd') else f32_wgrad_depth(kernel, n_out)


# dyadic probe operands: features {0, +-1, +-2} 2^-3, weights and gradients {0, +-1, +-2, +-3} 2^-4, so every product is a
# multiple of 2^-7 and an fp32 accumulation is exact in any order while sum |terms| < 2^24 x 2^-7
PROBE_X, PROBE_W, PROBE_GRID = (0., 1., -1., 2., -2.), (0., 1., -1., 2., -2., 3., -3.), 2.0 ** -7


def probe_values(shape, vals, scale, generator=None, device='cpu'):
    v = torch.tensor(vals, dtype=torch.float32, device=device) * scale
    return v[torch.randint(len(vals), shape, generator=generator, device=device)]


def probe_x(shape, generator=None, device='cpu'):
    return probe_values(shape, PROBE_X, 2.0 ** -3, generator, device)


def probe_w(shape, generator=None, device='cpu'):
    return probe_values(shape, PROBE_W, 2.0 ** -4, generator, device)


def binade_rows(n, c, spread=8, generator=None, device='cpu'):
    """random fp32 rows whose magnitudes span 2 spread + 1 binades (one power-of-two scale per row)"""
    x = torch.randn((n, c), generator=generator, device=device)
    e = torch.randint(-spread, spread + 1, (n, 1), generator=generator, device=device).float()
    return x * torch.exp2(e)


# ------------------------------------------------------------------ split rows
def split_halves(raw, c):
    """split rows (uint8 [n, 4c]) -> (hi, lo) bf16 [n, c]"""
    n = raw.shape[0]
    b = raw.contiguous().view(torch.bfloat16).view(n, c // 32, 2, 32)
    return b[:, :, 0].reshape(n, c), b[:, :, 1].reshape(n, c)


def split_decode(raw, c):
    """split rows -> fp64 hi + lo (exact)"""
    hi, lo = split_halves(raw, c)
    return hi.double() + lo.double()


def split_encode(hi, lo):
    """bf16 [n, c] halves -> split rows uint8 [n, 4c]"""
    n, c = hi.shape
    b = torch.stack([hi.reshape(n, c // 32, 32), lo.reshape(n, c // 32, 32)], 2)
    return b.reshape(n, 2 * c).contiguous().view(torch.uint8)


def split_of(v):
    """the documented split of fp32 values: hi = bf16_rn(v), lo = bf16_rn(v - hi)"""
    v = v.float()
    hi = v.bfloat16()
    return split_encode(hi, (v - hi.float()).bfloat16())


# ------------------------------------------------------------------ references
def conv(x, nbr, n_out, w, want_abs=True):
    """y[o] = sum_k x[nbr[k][o]] @ w[k]  (nbr None: identity, K == 1).  x fp64 [n_in, cin], w [K, cin, cout].
    Returns (y, A) in fp64 with A = sum_k |x[nbr]| @ |w[k]|."""
    w = w.double()
    y = torch.zeros((n_out, w.shape[2]), dtype=torch.float64, device=x.device)
    a = torch.zeros_like(y) if want_abs else None
    ax, aw = x.abs(), w.abs()
    if nbr is None:
        assert w.shape[0] == 1 and x.shape[0] == n_out
        return x @ w[0], (ax @ aw[0] if want_abs else None)
    nbr = nbr.long()
    for k in range(w.shape[0]):
        o = (nbr[k] >= 0).nonzero().squeeze(1)
        if o.numel():
            i = nbr[k][o]
            y.index_add_(0, o, x[i] @ w[k])
            if want_abs:
                a.index_add_(0, o, ax[i] @ aw[k])
    return y, a


def epilogue(y, a, scale=None, shift=None, res=None, relu=False):
    """y * scale + shift + res, ReLU; A scaled alike (|scale| A + |shift| + |res|)"""
    if scale is not None:
        y, a = y * scale.double(), a * scale.double().abs()
    if shift is not None:
        y, a = y + shift.double(), a + shift.double().abs()
    if res is not None:
        y, a = y + res, a + res.abs()
    if relu:
        y = torch.relu(y)
    return y, a


def convtr(x, down_nbr, w, n_fine):
    """dense transposed stride-2 convolution: out[down_nbr[k][o]] = x[o] @ w[k] (every fine row covered once).
    w [kvol, cin, cout].  Returns (y, A)."""
    w = w.double()
    kvol, n_coarse = down_nbr.shape
    y = torch.zeros((n_fine, w.shape[2]), dtype=torch.float64, device=x.device)
    a = torch.zeros_like(y)
    hits = torch.zeros(n_fine, dtype=torch.int64, device=x.device)
    d = down_nbr.long()
    for k in range(kvol):
        o = (d[k] >= 0).nonzero().squeeze(1)
        f = d[k][o]
        y[f] = x[o] @ w[k]
        a[f] = x[o].abs() @ w[k].abs()
        hits.index_add_(0, f, torch.ones_like(f))
    assert bool((hits == 1).all()), "dense transposed convolution: a fine row is not covered exactly once"
    return y, a


def transpose_map(nbr, n_in):
    """nbr_t[k][i] = o  iff  nbr[k][o] = i (else -1)"""
    K, n_out = nbr.shape
    t = torch.full((K, n_in), -1, dtype=torch.int64, device=nbr.device)
    for k in range(K):
        o = (nbr[k] >= 0).nonzero().squeeze(1)
        t[k, nbr[k][o].long()] = o
    return t


def _keys(c):
    c = c.long()
    return ((c[:, 0] << 54) | ((c[:, 1] + (1 << 17)) << 36) | ((c[:, 2] + (1 << 17)) << 18) | (c[:, 3] + (1 << 17)))


def neighbour_map(coords, ks, step):
    """Kernel map of an odd ks^3 kernel over one coordinate set (int32 [n, 4] rows (b, x, y, z)), found independently of
    the library: nbr[k][o] = row of coords[o] + delta_k * step, offsets x fastest, centred."""
    keys = _keys(coords)
    sk, order = torch.sort(keys)
    h = ks // 2
    out = []
    r = torch.arange(-h, h + 1, device=coords.device)
    for dz in r:
        for dy in r:
            for dx in r:
                q = coords.long().clone()
                q[:, 1] += int(dx) * step
                q[:, 2] += int(dy) * step
                q[:, 3] += int(dz) * step
                qk = _keys(q)
                pos = torch.searchsorted(sk, qk).clamp(max=len(sk) - 1)
                out.append(torch.where(sk[pos] == qk, order[pos], torch.full_like(pos, -1)))
    return torch.stack(out)


def wgrad(x, nbr, gout, K):
    """gw[k] = sum_o x[nbr[k][o]]^T gout[o] (nbr None: identity); returns (gw, A) fp64 [K, cin, cout]"""
    gw = torch.zeros((K, x.shape[1], gout.shape[1]), dtype=torch.float64, device=x.device)
    a = torch.zeros_like(gw)
    for k in range(K):
        if nbr is None:
            xi, g = x, gout
        else:
            o = (nbr[k] >= 0).nonzero().squeeze(1)
            xi, g = x[nbr[k][o].long()], gout[o]
        gw[k] = xi.t() @ g
        a[k] = xi.abs().t() @ g.abs()
    return gw, a


def worst(y, ref, a, c, split_out=False):
    """max over elements of |y - ref| / (2^-16 A [+ 2^-17 |ref| / c]) -- the fraction of 2^-16 A the error uses; the
    bound holds when this is <= c"""
    err = (y.double() - ref).abs()
    if split_out:
        err = (err - OUT_SPLIT * ref.abs()).clamp(min=0)
    a = a * 2.0 ** -16
    r = err / a.clamp(min=1e-300)
    r = torch.where((a == 0) & (err == 0), torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def exact_budget_bits(terms_abs_sum, grid):
    """log2 of (sum |terms| / grid): an fp32 accumulation of grid multiples is exact while this stays below 24"""
    m = float(terms_abs_sum.max()) if terms_abs_sum.numel() else 0.0
    return math.log2(m / grid) if m > 0 else 0.0
