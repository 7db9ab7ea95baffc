"""Host-side planning of the persistent convolution kernel (csrc/conv_chain.cu), checked without a GPU.

``osb_conv_desc_fill`` / ``osb_conv_chain_workspace_bytes`` are pure host functions: they choose the tile shape, the
split factor and the stage partition of a layer and validate the arguments.  The kernel then derives every role's loop
from those few integers, so the invariants below are what keeps the roles (weight producer, gather warps, two consumer
warpgroups) walking the same sequence of items: a violation would be a hang or a silently skipped unit on the device.
The walk itself (``_items``) restates the kernel's ``CH_FOR_ITEMS`` macro; the descriptor numbers come from the library."""
import ctypes
import struct

import pytest

from openscene_b200 import _cabi as C

FAKE = 0x10000            # any non-NULL, 256-byte aligned address: the descriptor is only filled, never launched

# ConvDesc (csrc/conv_chain.cu): 12 pointers, int64 n_out, 14 int32, 8 x int32 padding = 192 bytes
_FMT = '<12Q q 14i 8i'
_INTS = ('K', 'nb0', 'nb1', 'cout', 'cout_pad', 'nt', 'n_ntiles', 'relu', 'cmap_cout', 'nsplit', 'm_tiles', 'nsub_max',
         'barrier_before', 'stages_per_split')


def _fill(n_out, K, c0, c1, cout, *, cmap=0, cmap_cout=0, ws=None, barrier=0, res=0, nbr=FAKE, out_split=FAKE, out_f32=0,
          scale=0, shift=0):
    L = C.lib()
    assert struct.calcsize(_FMT) == L.osb_conv_desc_bytes() == 192
    buf = ctypes.create_string_buffer(192)
    need = 0 if cmap else L.osb_conv_chain_workspace_bytes(n_out, K, c0 + c1, cout)
    if ws is None:
        ws = (FAKE, need) if need else (0, 0)
    rc = L.osb_conv_desc_fill(ctypes.addressof(buf), FAKE, c0, FAKE if c1 else None, c1, nbr or None, n_out, K, FAKE, cout,
                              scale or None, shift or None, res or None, 1, out_split or None, out_f32 or None, None,
                              cmap or None, cmap_cout, ws[0] or None, ws[1], barrier)
    if rc:
        return None, (L.osb_last_error() or b'').decode()
    v = struct.unpack(_FMT, buf.raw)
    d = dict(zip(_INTS, v[13:27]))
    d['n_out'], d['partial'], d['need'] = v[12], v[11], need
    return d, ''


def _items(d, grid):
    """The kernel's CH_FOR_ITEMS for every CTA: [(cta, z, n_tile, m, nsub, t_begin, t_end)]."""
    T = d['K'] * (d['nb0'] + d['nb1'])
    per_z = d['m_tiles'] * d['n_ntiles']
    U = per_z * d['nsplit']
    out = []
    for cta in range(grid):
        u, u_end = U * cta // grid, U * (cta + 1) // grid
        while u < u_end:
            z, r = divmod(u, per_z)
            nti, m = divmod(r, d['m_tiles'])
            nsub = 2 if (d['nsub_max'] == 2 and u + 1 < u_end and m + 1 < d['m_tiles']) else 1
            t_begin = min(z * d['stages_per_split'], T)
            out.append((cta, z, nti, m, nsub, t_begin, min(t_begin + d['stages_per_split'], T)))
            u += nsub
    return out


# (rows, K, cin0, cin1, cout): every layer shape of MinkUNet18A/34C on the bench scene, the lidar scene, and edge sizes
SHAPES = [(197382, 27, 96, 0, 96), (197382, 27, 96, 32, 96), (197382, 1, 96, 32, 96), (197382, 1, 96, 0, 768),
          (40640, 27, 32, 0, 32), (40640, 8, 32, 0, 32), (40640, 27, 128, 64, 128), (9674, 27, 64, 0, 64),
          (9674, 27, 256, 128, 128), (2136, 27, 128, 0, 128), (2136, 27, 256, 128, 256), (473, 27, 256, 0, 256),
          (473, 1, 128, 0, 256), (473, 8, 128, 0, 256), (1023329, 27, 96, 32, 96), (74511, 27, 256, 0, 256),
          (1, 27, 32, 0, 32), (127, 27, 32, 0, 32), (128, 1, 32, 0, 32), (129, 27, 64, 0, 96), (5000, 27, 32, 0, 160),
          (300, 27, 256, 0, 512), (70000, 1, 96, 0, 512)]


@pytest.mark.parametrize('n_out,K,c0,c1,cout', SHAPES)
def test_descriptor_invariants(n_out, K, c0, c1, cout):
    d, err = _fill(n_out, K, c0, c1, cout)
    assert d is not None, err
    T = K * (c0 + c1) // 32
    assert (d['K'], d['nb0'], d['nb1'], d['cout'], d['n_out']) == (K, c0 // 32, c1 // 32, cout, n_out)
    # tile shape: the padded width is whole N tiles of at most 128 columns; two row tiles share a weight tile only when the
    # N tile is at most 64 wide (a consumer thread then holds at most 64 fp32 accumulators)
    assert d['cout_pad'] >= cout and d['cout_pad'] == d['nt'] * d['n_ntiles'] and d['nt'] <= 128 and d['nt'] % 16 == 0
    assert d['nsub_max'] == (2 if d['nt'] <= 64 else 1)
    assert d['m_tiles'] == -(-n_out // 128)
    # stage partition: splits tile [0, T) without an empty one
    ns, sps = d['nsplit'], d['stages_per_split']
    assert 1 <= ns <= 32 and ns * sps >= T and (ns - 1) * sps < T
    # scratch: the query is an upper bound of what the fill demands (it is made before empty splits are dropped)
    used = ns * n_out * d['cout_pad'] * 4 if ns > 1 else 0
    assert used <= d['need'] <= 32 * n_out * d['cout_pad'] * 4 and (d['need'] > 0) == (ns > 1)
    assert (d['partial'] != 0) == (ns > 1)


@pytest.mark.parametrize('n_out,K,c0,c1,cout', SHAPES)
@pytest.mark.parametrize('grid', [148, 132, 7])
def test_every_unit_is_visited_exactly_once(n_out, K, c0, c1, cout, grid):
    d, err = _fill(n_out, K, c0, c1, cout)
    assert d is not None, err
    T = K * (c0 + c1) // 32
    seen = {}
    for (cta, z, nti, m, nsub, t0, t1) in _items(d, grid):
        assert 0 <= z < d['nsplit'] and 0 <= nti < d['n_ntiles'] and t0 < t1 <= T          # no empty item: accFull would never fire
        for s in range(nsub):
            assert m + s < d['m_tiles']                                                       # both sub-tiles inside the same N tile / split
            key = (z, nti, m + s)
            assert key not in seen
            seen[key] = (t0, t1)
    assert len(seen) == d['m_tiles'] * d['n_ntiles'] * d['nsplit']
    # per (row tile, N tile) the splits cover every stage exactly once, in order (fixed-order reduction)
    for nti in range(d['n_ntiles']):
        for m in (0, d['m_tiles'] - 1):
            spans = [seen[(z, nti, m)] for z in range(d['nsplit'])]
            assert spans[0][0] == 0 and spans[-1][1] == T
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def test_split_factor_rules():
    """Splitting exists for the levels with few tiles per SM (the cost model may still pick 2 for a level of ~2 waves); the
    full-resolution layers are never split."""
    for (n_out, K, c0, c1, cout) in SHAPES:
        d, _ = _fill(n_out, K, c0, c1, cout)
        tiles = d['m_tiles'] * d['n_ntiles']
        if tiles >= 4 * 148:
            assert d['nsplit'] == 1, (n_out, K, c0, c1, cout)
        if K * (c0 + c1) // 32 == 1:
            assert d['nsplit'] == 1
    d, _ = _fill(473, 27, 256, 0, 256)            # 8 tiles x 216 stages: split as far as the cap allows
    assert d['nsplit'] >= 16
    L = C.lib()
    assert L.osb_tuning_set(b'chain_force_split', 1) == 0
    try:
        d1, _ = _fill(473, 27, 256, 0, 256)
        assert d1['nsplit'] == 1 and d1['need'] == 0
    finally:
        assert L.osb_tuning_set(b'chain_force_split', 0) == 0
    assert L.osb_tuning_set(b'no_such_knob', 1) != 0 and b'unknown knob' in L.osb_last_error()


def test_dense_transposed_form():
    d, err = _fill(40640, 1, 128, 0, 8 * 96, cmap=FAKE, cmap_cout=96, nbr=0)
    assert d is not None, err
    assert d['nsplit'] == 1 and d['cmap_cout'] == 96 and d['cout_pad'] == 768 and d['nt'] == 128 and d['n_ntiles'] == 6


@pytest.mark.parametrize('kw,msg', [
    (dict(n_out=100, K=27, c0=48, c1=0, cout=32), 'multiples of 32'),
    (dict(n_out=100, K=27, c0=32, c1=0, cout=20), 'multiple of 32'),
    (dict(n_out=100, K=64, c0=32, c1=0, cout=32), 'not supported'),
    (dict(n_out=0, K=27, c0=32, c1=0, cout=32), 'bad row count'),
    (dict(n_out=1 << 31, K=1, c0=32, c1=0, cout=32), 'bad row count'),
    (dict(n_out=100, K=27, c0=32, c1=0, cout=32, nbr=0), 'identity map needs K == 1'),
    (dict(n_out=100, K=27, c0=32, c1=0, cout=32, out_split=0), 'no output'),
    (dict(n_out=100, K=27, c0=32, c1=0, cout=32, scale=FAKE), 'scale and shift'),
    (dict(n_out=100, K=1, c0=32, c1=0, cout=1024), 'output channels per row'),
    (dict(n_out=100, K=1, c0=32, c1=0, cout=256, cmap=FAKE, cmap_cout=96), 'dense-transpose'),
    (dict(n_out=100, K=1, c0=32, c1=0, cout=256, cmap=FAKE, cmap_cout=64, res=FAKE), 'dense-transpose'),
    (dict(n_out=473, K=27, c0=256, c1=0, cout=256, ws=(FAKE, 1024)), 'workspace of'),
    (dict(n_out=473, K=27, c0=256, c1=0, cout=256, ws=(0, 0)), 'workspace of'),
])
def test_bad_arguments_fail_loudly(kw, msg):
    d, err = _fill(kw.pop('n_out'), kw.pop('K'), kw.pop('c0'), kw.pop('c1'), kw.pop('cout'), **kw)
    assert d is None and msg in err, err


def test_launch_refuses_inconsistent_chains_before_touching_the_device():
    """osb_conv_chain_launch validates the layer list on the host first: these calls return an error without a GPU."""
    L = C.lib()
    assert L.osb_conv_chain_launch(None, 1, None, 0, None) != 0
    buf = ctypes.create_string_buffer(2 * 192)
    # first layer of a launch asking for a grid barrier
    rc = L.osb_conv_desc_fill(ctypes.addressof(buf), FAKE, 32, None, 0, FAKE, 1000, 1, FAKE, 32, None, None, None, 1, FAKE, None,
                              None, None, 0, None, 0, 1)     # K = 1: one stage, never split
    assert rc == 0
    assert L.osb_conv_chain_launch(ctypes.addressof(buf), 1, FAKE, 0, None) != 0
    assert b'first layer' in L.osb_last_error()
    # two split layers back to back on the same scratch without a barrier between them
    need = L.osb_conv_chain_workspace_bytes(473, 27, 256, 256)
    assert need > 0
    for i in range(2):
        rc = L.osb_conv_desc_fill(ctypes.addressof(buf) + 192 * i, FAKE, 256, None, 0, FAKE, 473, 27, FAKE, 256, None, None, None, 1,
                                  FAKE, None, None, None, 0, FAKE, need, 0)
        assert rc == 0
    assert L.osb_conv_chain_launch(ctypes.addressof(buf), 2, FAKE, 0, None) != 0
    assert b'share a split workspace' in L.osb_last_error()


def test_size_queries_survive_degenerate_shapes():
    """A size query is called before the arguments are validated (the caller needs the scratch to make the call): shapes the
    launch functions reject must come back as 0, not as a division by zero inside the library."""
    L = C.lib()
    for fn in (L.osb_conv_chain_workspace_bytes, L.osb_conv_tc_workspace_bytes, L.osb_conv_wgrad_tc_workspace_bytes):
        for (n, K, cin, cout) in [(0, 27, 32, 32), (-5, 27, 32, 32), (100, 0, 32, 32), (100, 27, 0, 32), (100, 27, 16, 32),
                                  (100, 27, 32, 0)]:
            assert fn(n, K, cin, cout) == 0
    assert L.osb_coordset_workspace_bytes(0) >= 0 and L.osb_voxelize_workspace_bytes(0) >= 0
    assert L.osb_feature_remap_workspace_bytes(0, 0) >= 0 and L.osb_fusion_workspace_bytes(0, 0) >= 0
