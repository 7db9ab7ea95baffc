"""csrc/pool.cu through the C ABI against the NumPy restatement (tests/pool_ref.py), bit for bit: local sum / average / max
forward and backward over real kernel maps (K = 1, 8, 27, 125, strides 1 and 2, dilation 2, negative coordinates) and over
synthetic maps with row counts either side of every tile edge of the launch plan; global sum / average / max with exact
probes, interleaved batch rows, empty batch indices and the grown-chunk plan.  Outputs go into NaN-filled buffers, every
launch runs twice and must give the same bits, and every host refusal is exercised."""
import ctypes

import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import synth
from tests import pool_ref as P

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float('nan'), dtype=dtype, device=DEV)


def _fwd(x, nbr, mode):
    n_out, c = nbr.shape[1], x.shape[1]
    out = _nan((n_out, c))
    count = torch.full((n_out,), -7, dtype=torch.int32, device=DEV)
    argk = torch.full((n_out, c), 0x1234, dtype=torch.int16, device=DEV)
    C.call('osb_pool_fwd', C.ptr(x), c, C.ptr(nbr), n_out, nbr.shape[0], mode, C.ptr(out), C.ptr(count), C.ptr(argk),
           C.stream_ptr())
    return out, count, argk


def _bwd(g, nbr_t, mode, count, argk):
    n_in, c = nbr_t.shape[1], g.shape[1]
    gin = _nan((n_in, c))
    C.call('osb_pool_bwd', C.ptr(g), c, C.ptr(nbr_t), n_in, nbr_t.shape[0], mode, C.ptr(count), C.ptr(argk), C.ptr(gin),
           C.stream_ptr())
    return gin


def _bits(t):
    """fp32 bit patterns with every NaN mapped to one pattern (the payload of a NaN made by inf - inf is not specified)"""
    a = np.array(t.cpu().numpy() if torch.is_tensor(t) else t, np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7fc00000
    return b


def _values(shape, seed, special=False):
    """random fp32 (not dyadic); with special: ties, +-0, +-inf and NaN mixed in"""
    rng = np.random.RandomState(seed)
    x = (rng.randn(*shape) * 4).astype(np.float32)
    if special:
        pool = np.array([0.0, -0.0, 1.0, 1.0, np.inf, -np.inf, np.nan, -3.0], np.float32)
        m = rng.rand(*shape) < 0.3
        x[m] = pool[rng.randint(len(pool), size=int(m.sum()))]
    return x


def _check_local(x_np, nbr_np, modes=(P.SUM, P.AVG, P.MAX), seed=0):
    n_in = x_np.shape[0]
    x = torch.from_numpy(x_np).to(DEV)
    nbr = torch.from_numpy(np.ascontiguousarray(nbr_np, np.int32)).to(DEV)
    nbr_t_np = P.transpose_map(nbr_np, n_in)
    nbr_t = torch.from_numpy(nbr_t_np).to(DEV)
    g_np = _values((nbr_np.shape[1], x_np.shape[1]), seed + 1)
    g = torch.from_numpy(g_np).to(DEV)
    for mode in modes:
        out, cnt, win = P.pool_fwd(x_np, nbr_np, mode)
        o1, c1, a1 = _fwd(x, nbr, mode)
        o2, c2, a2 = _fwd(x, nbr, mode)
        assert np.array_equal(_bits(o1), _bits(out)), f"mode {mode} forward"
        assert torch.equal(o1.view(torch.int32), o2.view(torch.int32))
        if mode == P.AVG:
            assert np.array_equal(c1.cpu().numpy(), cnt) and torch.equal(c1, c2)
        if mode == P.MAX:
            assert np.array_equal(a1.cpu().numpy().view(np.uint16), win) and torch.equal(a1, a2)
        gin = P.pool_bwd(g_np, nbr_np, mode, cnt, win, n_in)
        b1 = _bwd(g, nbr_t, mode, c1, a1)
        b2 = _bwd(g, nbr_t, mode, c1, a1)
        assert np.array_equal(_bits(b1), _bits(gin)), f"mode {mode} backward"
        assert torch.equal(b1.view(torch.int32), b2.view(torch.int32))


def _real_map(n, extent, ks, stride, dil, seed, batch=2, offset=0):
    from openscene_b200.coords import CoordinateManager
    cl = synth.random_cloud(n, extent, seed=seed, batch=batch)
    cl[:, 1:] -= offset
    cm = CoordinateManager(torch.from_numpy(cl).to(DEV))
    ts_out = cm.stride(1, stride) if stride > 1 else 1
    km = cm.kernel_map(1, ts_out, ks, dil)
    return km.nbr.cpu().numpy(), cm.sets[1].n


@pytest.mark.parametrize('ks,stride,dil,offset', [(1, 2, 1, 0), (2, 2, 1, 0), (3, 1, 1, 0), (3, 2, 1, 9), (5, 1, 1, 0),
                                                  (3, 1, 2, 0), (2, 2, 1, 13)])
@pytest.mark.parametrize('c', [1, 3, 20, 32, 96, 256, 257])
def test_local_pooling_on_kernel_maps(ks, stride, dil, offset, c):
    nbr, n_in = _real_map(700 if c > 96 else 1500, 14, ks, stride, dil, seed=ks * 7 + c, offset=offset)
    _check_local(_values((n_in, c), c + ks, special=(c in (3, 32))), nbr, seed=c)


def _synthetic_map(n_in, n_out, K, density, seed):
    """an injective partial map per offset, like a convolution's"""
    rng = np.random.RandomState(seed)
    nbr = np.full((K, n_out), -1, np.int64)
    for k in range(K):
        o = np.nonzero(rng.rand(n_out) < density)[0][:n_in]
        nbr[k, o] = rng.permutation(n_in)[:len(o)]
    return nbr


def _tile_rows(c):
    """rows per block of the local launch plan (lanes = channel groups rounded up to a power of two, at most 64) and rows per
    full grid pass (132 * 16 blocks)"""
    lanes = 1
    while lanes < (c + 3) // 4 and lanes < 64:
        lanes *= 2
    rpb = 256 // lanes
    return rpb, rpb * 132 * 16


@pytest.mark.parametrize('c', [1, 3, 20, 32, 96, 256, 257])
def test_local_pooling_either_side_of_tile_edges(c):
    rpb, rpg = _tile_rows(c)
    for n_out in sorted({1, rpb - 1, rpb, rpb + 1, 2 * rpb + 1}):
        if n_out < 1:
            continue
        nbr = _synthetic_map(n_out + 5, n_out, 8, 0.7, seed=n_out)
        _check_local(_values((n_out + 5, c), n_out, special=True), nbr, seed=n_out)
    for n_out in (rpg - 1, rpg + 1):                                   # one offset: the grid-stride loop's second pass
        nbr = _synthetic_map(n_out, n_out, 1, 0.9, seed=3)
        _check_local(_values((n_out, c), 4), nbr, modes=(P.MAX,) if c > 32 else (P.SUM, P.AVG, P.MAX))


def test_max_edge_cases_through_the_kernel():
    """ties to the lowest k, the first NaN, +-0, +-inf, windows with no present input (0, no winner, no gradient)"""
    x = np.array([[1], [3], [3], [2], [np.nan], [5], [np.nan], [-0.0], [0.0], [-np.inf], [-np.inf], [7]], np.float32)
    nbr = np.array([[0, 4, 7, 9, -1, 11], [1, 5, 8, 10, -1, -1], [2, 6, -1, -1, -1, -1], [3, -1, -1, -1, -1, -1]])
    _check_local(x, nbr, seed=5)
    _, _, win = _fwd(torch.from_numpy(x).to(DEV), torch.from_numpy(nbr.astype(np.int32)).to(DEV), P.MAX)
    assert win.cpu().numpy().view(np.uint16)[:, 0].tolist() == [1, 0, 0, 0, P.NO_WINNER, 0]


def test_k_65535_uses_every_winner_code():
    n = 3
    nbr = np.full((65535, n), -1, np.int64)
    nbr[65534, 0], nbr[0, 1], nbr[65533, 2] = 0, 1, 2
    _check_local(_values((n, 4), 1), nbr, seed=2)


# ------------------------------------------------------------------ global
def _gfwd(x, batch, n_batch, mode):
    n, c = x.shape
    out = _nan((n_batch, c))
    count = torch.full((n_batch,), -7, dtype=torch.int32, device=DEV)
    argrow = torch.full((n_batch, c), -9, dtype=torch.int32, device=DEV)
    wsb = C.lib().osb_global_pool_workspace_bytes(n, c, n_batch)
    ws = torch.full((wsb,), 0x5A, dtype=torch.uint8, device=DEV)
    C.call('osb_global_pool_fwd', C.ptr(x), C.ptr(batch), n, c, n_batch, mode, C.ptr(out), C.ptr(count), C.ptr(argrow),
           C.ptr(ws), wsb, C.stream_ptr())
    return out, count, argrow


def _gbwd(g, batch, n, mode, count, argrow):
    gin = _nan((n, g.shape[1]))
    C.call('osb_global_pool_bwd', C.ptr(g), C.ptr(batch), n, g.shape[1], mode, C.ptr(count), C.ptr(argrow), C.ptr(gin),
           C.stream_ptr())
    return gin


def _check_global(x_np, batch_np, n_batch, exact, seed=0):
    n, c = x_np.shape
    x = torch.from_numpy(x_np).to(DEV)
    batch = torch.from_numpy(batch_np.astype(np.int32)).to(DEV)
    g_np = _values((n_batch, c), seed)
    g = torch.from_numpy(g_np).to(DEV)
    for mode in (P.SUM, P.AVG, P.MAX):
        ref, cnt, arg = P.global_fwd_exact(x_np, batch_np, n_batch, mode)
        o1, c1, a1 = _gfwd(x, batch, n_batch, mode)
        o2, c2, a2 = _gfwd(x, batch, n_batch, mode)
        assert torch.equal(o1.view(torch.int32), o2.view(torch.int32)), mode
        if mode == P.MAX or exact:
            assert np.array_equal(_bits(o1), _bits(ref)), mode
        else:
            r64, bound = P.global_sum_bound(x_np, batch_np, n_batch, mode)
            got = o1.cpu().numpy().astype(np.float64)
            fin = np.isfinite(r64)
            assert np.all(np.abs(got[fin] - r64[fin]) <= bound[fin]), mode
            assert np.array_equal(np.isnan(got), np.isnan(r64))
        if mode == P.AVG:
            assert np.array_equal(c1.cpu().numpy(), cnt)
        if mode == P.MAX:
            assert np.array_equal(a1.cpu().numpy(), arg) and torch.equal(a1, a2)
        gin = P.global_bwd(g_np, batch_np, mode, cnt, arg)
        b1 = _gbwd(g, batch, n, mode, c1, a1)
        assert np.array_equal(_bits(b1), _bits(gin)), mode
        assert torch.equal(b1.view(torch.int32), _gbwd(g, batch, n, mode, c1, a1).view(torch.int32))


def _dyadic(shape, seed):
    rng = np.random.RandomState(seed)
    return (rng.randint(-64, 65, size=shape) * 2.0 ** rng.randint(-8, 3, size=shape)).astype(np.float32)


@pytest.mark.parametrize('n', [1, 255, 256, 257, 513, 3000])
@pytest.mark.parametrize('c', [1, 3, 32, 257])
def test_global_pooling_exact_probes(n, c):
    rng = np.random.RandomState(n + c)
    for n_batch, interleave in ((1, False), (3, False), (3, True)):
        b = np.sort(rng.randint(0, n_batch, size=n)) if not interleave else rng.randint(0, n_batch, size=n)
        _check_global(_dyadic((n, c), n), b, n_batch + (1 if interleave else 0), exact=True, seed=c)


def test_global_pooling_bounds_and_special_values():
    n, c = 5000, 20
    rng = np.random.RandomState(0)
    b = rng.randint(0, 4, size=n)
    _check_global(_values((n, c), 1), b, 5, exact=False)
    x = _values((n, c), 2, special=True)
    x[:, :3] = np.where(np.isnan(x[:, :3]), 0, x[:, :3])
    ref, _, arg = P.global_fwd_exact(x, b, 5, P.MAX)
    out, _, a = _gfwd(torch.from_numpy(x).to(DEV), torch.from_numpy(b.astype(np.int32)).to(DEV), 5, P.MAX)
    assert np.array_equal(_bits(out), _bits(ref)) and np.array_equal(a.cpu().numpy(), arg)


def test_global_pooling_with_grown_chunks():
    """1024 batch indices x 257 channels: the partial slots would exceed the workspace budget at 256-row chunks"""
    n, c, nb = 10000, 257, 1024
    rng = np.random.RandomState(3)
    _check_global(_dyadic((n, c), 5), rng.randint(0, nb, size=n), nb, exact=True)


# ------------------------------------------------------------------ host refusals
def _rc(name, *args):
    rc = getattr(C.lib(), name)(*args)
    return rc, (C.lib().osb_last_error() or b'').decode()


def test_host_refusals():
    x = torch.zeros(8, 4, device=DEV)
    nbr = torch.zeros(2, 8, dtype=torch.int32, device=DEV)
    out = torch.zeros(8, 4, device=DEV)
    cnt = torch.zeros(8, dtype=torch.int32, device=DEV)
    ak = torch.zeros(8, 4, dtype=torch.int16, device=DEV)
    s = C.stream_ptr()
    p = C.ptr
    for fn in ('osb_pool_fwd', 'osb_pool_bwd'):
        # fwd (in, c, nbr, n_out, K, mode, out, count, argk, stream); bwd (gout, c, nbr_t, n_in, K, mode, count, argk, gin, stream)
        ok = (p(x), 4, p(nbr), 8, 2, 0, p(out), p(cnt), p(ak), s) if fn == 'osb_pool_fwd' else \
            (p(x), 4, p(nbr), 8, 2, 0, p(cnt), p(ak), p(out), s)
        i_cnt, i_ak = (7, 8) if fn == 'osb_pool_fwd' else (6, 7)
        i_out = 6 if fn == 'osb_pool_fwd' else 8
        assert _rc(fn, *ok)[0] == 0
        for i, v, msg in ((5, 3, 'bad mode'), (5, -1, 'bad mode'), (4, 0, 'outside'), (4, 65536, 'outside'),
                          (1, 0, 'bad shape'), (3, 0, 'bad shape'), (0, None, 'NULL'), (2, None, 'NULL'),
                          (i_out, None, 'NULL')):
            a = list(ok)
            a[i] = v
            rc, err = _rc(fn, *a)
            assert rc != 0 and msg in err, (fn, i, v, err)
        a = list(ok)
        a[5], a[i_cnt] = 1, None
        rc, err = _rc(fn, *a)
        assert rc != 0 and 'count' in err                                   # avg without counts
        a = list(ok)
        a[5], a[i_ak] = 2, None
        rc, err = _rc(fn, *a)
        assert rc != 0 and 'winner' in err                                  # max without winners
        a = list(ok)
        a[i_cnt], a[i_ak] = None, None
        assert _rc(fn, *a)[0] == 0                                          # sum needs neither
    torch.cuda.synchronize()
    b = torch.zeros(8, dtype=torch.int32, device=DEV)
    g = torch.zeros(2, 4, device=DEV)
    ar = torch.zeros(2, 4, dtype=torch.int32, device=DEV)
    wsb = C.lib().osb_global_pool_workspace_bytes(8, 4, 2)
    assert wsb > 0 and C.lib().osb_global_pool_workspace_bytes(0, 4, 2) == 0
    assert C.lib().osb_global_pool_workspace_bytes(8, -1, 2) == 0 and C.lib().osb_global_pool_workspace_bytes(8, 4, 0) == 0
    ws = torch.zeros(wsb + 16, dtype=torch.uint8, device=DEV)
    ok = [p(x), p(b), 8, 4, 2, 0, p(g), p(cnt), p(ar), p(ws), wsb, s]
    assert _rc('osb_global_pool_fwd', *ok)[0] == 0
    for i, v, msg in ((5, 7, 'bad mode'), (2, 0, 'bad shape'), (3, 0, 'bad shape'), (4, 0, 'bad shape'), (0, None, 'NULL'),
                      (1, None, 'NULL'), (6, None, 'NULL'), (9, None, 'workspace'), (10, wsb - 1, 'workspace'),
                      (9, ctypes.c_void_p(ws.data_ptr() + 4), 'aligned')):
        a = list(ok)
        a[i] = v
        rc, err = _rc('osb_global_pool_fwd', *a)
        assert rc != 0 and msg in err, (i, v, err)
    for mode, i in ((1, 7), (2, 8)):
        a = list(ok)
        a[5], a[i] = mode, None
        assert _rc('osb_global_pool_fwd', *a)[0] != 0
    okb = [p(g), p(b), 8, 4, 0, p(cnt), p(ar), p(x), s]
    assert _rc('osb_global_pool_bwd', *okb)[0] == 0
    for i, v, msg in ((4, 3, 'bad mode'), (2, 0, 'bad shape'), (3, 0, 'bad shape'), (0, None, 'NULL'), (1, None, 'NULL'),
                      (7, None, 'NULL')):
        a = list(okb)
        a[i] = v
        rc, err = _rc('osb_global_pool_bwd', *a)
        assert rc != 0 and msg in err, (i, v, err)
    for mode, i in ((1, 5), (2, 6)):
        a = list(okb)
        a[4], a[i] = mode, None
        assert _rc('osb_global_pool_bwd', *a)[0] != 0
    torch.cuda.synchronize()
