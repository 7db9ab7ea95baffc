"""tests/norm_ref.py without a GPU: the fp64 references against torch's own train-mode BatchNorm and cross-entropy, simulated
kernel evaluation orders (the launch plan's blocks, row slots and merges, fp32 roundings of the outputs, the apply pass in fp32
with and without FMA contraction) inside the bounds, the probe generators inside their exactness budget, and negative
controls -- each a plausible kernel or wiring mistake -- that must break a bound or an exact comparison."""
import pytest
import torch
import torch.nn.functional as F

from tests import norm_ref as NR
from tests import replay_ref as R


def _rows(n, c, seed, far=1000.0):
    g = torch.Generator().manual_seed(seed)
    sigma = torch.exp(8 * torch.rand(c, generator=g) - 4).double()
    mean = sigma * (2 * far * torch.rand(c, generator=g).double() - far)
    x = (mean + sigma * R.binade_rows(n, c, spread=3, generator=g).double()).float().double()
    w = (0.5 + torch.rand(c, generator=g)) * torch.where(torch.rand(c, generator=g) < 0.3, -1.0, 1.0)
    w[0] = 0.0
    b = torch.rand(c, generator=g) - 0.5
    return x, w, b, g


def _simulated_stats(x, w, b, eps):
    """the kernels' order: per block, 32 row slots each summing every 32nd row in fp64; slot merge; finalize with 8 slots
    over blocks and an 8-slot merge; then the finalize arithmetic and fp32 stores"""
    n, c = x.shape
    nblk, rpb = NR.bn_row_blocks(n), NR.bn_block_rows(n)
    d = x - x[0]
    part1, part2 = torch.zeros(nblk, c, dtype=torch.float64), torch.zeros(nblk, c, dtype=torch.float64)
    for blk in range(nblk):
        r0, r1 = blk * rpb, min(n, blk * rpb + rpb)
        a1 = torch.zeros(NR.BN_ROW_SLOTS, c, dtype=torch.float64)
        a2 = torch.zeros_like(a1)
        for base in range(r0, r1, NR.BN_ROW_SLOTS):
            blk_rows = d[base:min(r1, base + NR.BN_ROW_SLOTS)]
            k = blk_rows.shape[0]
            a1[:k] += blk_rows
            a2[:k] += blk_rows * blk_rows
        s1, s2 = torch.zeros(c, dtype=torch.float64), torch.zeros(c, dtype=torch.float64)
        for i in range(NR.BN_ROW_SLOTS):
            s1, s2 = s1 + a1[i], s2 + a2[i]
        part1[blk], part2[blk] = s1, s2
    m1, m2 = torch.zeros(8, c, dtype=torch.float64), torch.zeros(8, c, dtype=torch.float64)
    for blk in range(nblk):
        m1[blk % 8] += part1[blk]
        m2[blk % 8] += part2[blk]
    t1, t2 = torch.zeros(c, dtype=torch.float64), torch.zeros(c, dtype=torch.float64)
    for i in range(8):
        t1, t2 = t1 + m1[i], t2 + m2[i]
    dm = t1 / n
    v = t2 / n - dm * dm
    var = torch.where(v < 0, torch.zeros_like(v), v)
    mean = x[0] + dm
    istd = 1.0 / torch.sqrt(var + eps)
    sc = w.double() * istd
    return dict(mean=NR.f32(mean), invstd=NR.f32(istd), scale=NR.f32(sc), shift=NR.f32(b.double() - mean * sc),
                mean64=mean, var64=var)


# ---------------------------------------------------------------------------------------------------------------- references
def test_references_match_torch_batch_norm_autograd():
    x, w, b, g = _rows(300, 64, seed=1, far=10.0)
    rm, rv = torch.rand(64, dtype=torch.float64), 0.5 + torch.rand(64, dtype=torch.float64)
    st = NR.bn_stats(x, w, b, 1e-5)
    for momentum, nbt in ((0.1, 3), (None, 3)):
        rm_t, rv_t = rm.clone(), rv.clone()
        m = 1.0 / (nbt + 1) if momentum is None else momentum
        F.batch_norm(x, rm_t, rv_t, w.double(), b.double(), training=True, momentum=m, eps=1e-5)
        rm_r, rv_r, tracked, m_r = NR.bn_running(rm, rv, nbt, st, momentum)
        assert tracked == nbt + 1 and m_r == m
        assert torch.allclose(rm_r, rm_t, rtol=1e-13, atol=1e-13) and torch.allclose(rv_r, rv_t, rtol=1e-13, atol=0)
    _, smean, sinv = torch.ops.aten.native_batch_norm(x, w.double(), b.double(), None, None, True, 0.1, 1e-5)
    assert torch.allclose(st['mean'], smean, rtol=1e-13) and torch.allclose(st['invstd'], sinv, rtol=1e-12)
    r = torch.randn(300, 64, generator=g, dtype=torch.float64)
    rst = NR.bn_stats(r, torch.ones(64), torch.zeros(64), 1e-5)
    gin = torch.randn(300, 64, generator=g, dtype=torch.float64)
    for form in ('none', 'identity', 'normalised'):
        for relu in (True, False):
            xx, ww, bb = x.clone().requires_grad_(), w.double().requires_grad_(), b.double().requires_grad_()
            t = F.batch_norm(xx, None, None, ww, bb, training=True, eps=1e-5)
            rr = 0 if form == 'none' else (r if form == 'identity' else F.batch_norm(r, None, None, training=True, eps=1e-5))
            yy = torch.relu(t + rr) if relu else t + rr
            yy.backward(gin)
            y, _ = NR.bn_apply(x, st, None if form == 'none' else r, rst if form == 'normalised' else None, relu)
            assert torch.allclose(y, yy.detach(), rtol=1e-12, atol=1e-12)
            bw = NR.bn_backward(y if relu else None, gin, x, st['mean'], st['invstd'], w)
            assert torch.allclose(bw['t1'], bb.grad, rtol=1e-12, atol=1e-12)
            assert torch.allclose(bw['t2'], ww.grad, rtol=1e-12, atol=1e-12)
            dz, _ = NR.bn_dz(bw, torch.cat([bw['t1'], bw['t2']]))
            assert torch.allclose(dz, xx.grad, rtol=1e-10, atol=1e-12)


def test_relu_mask_follows_torch_threshold_backward():
    y = torch.tensor([[1.0, 0.0, -1.0, float('nan')]], dtype=torch.float64)
    bw = NR.bn_backward(y, torch.ones_like(y), torch.zeros_like(y), torch.zeros(4), torch.ones(4), torch.ones(4))
    t = y.clone().requires_grad_()
    torch.relu(t).backward(torch.ones_like(t))
    assert torch.equal(bw['gp'], t.grad) and torch.equal(bw['gp'], torch.tensor([[1.0, 0.0, 0.0, 1.0]], dtype=torch.float64))
    assert torch.isnan(NR.relu_nan(torch.tensor([float('nan')]))).all()


@pytest.mark.parametrize('ignore', [255, -100])
def test_ce_reference_matches_torch(ignore):
    g = torch.Generator().manual_seed(3)
    n, cin, c = 500, 64, 37
    x = torch.randn(n, cin, generator=g, dtype=torch.float64)
    w = torch.randn(cin, c, generator=g)
    perm = torch.randperm(n, generator=g).to(torch.int32)
    lab = torch.randint(0, c, (n,), generator=g)
    lab[torch.rand(n, generator=g) < 0.2] = ignore
    fw = NR.ce_forward(x, w, perm, lab, ignore)
    xx, ww = x.clone().requires_grad_(), w.double().requires_grad_()
    z = xx @ ww
    lab_int = lab[perm.long()]
    loss = F.cross_entropy(z, lab_int, ignore_index=ignore)
    (0.5 * loss).backward()
    assert abs(float(fw['loss']) - float(loss.detach())) < 1e-12
    assert fw['n_valid'] == int((lab != ignore).sum())
    assert torch.equal(fw['pred'][perm.long()], z.detach().argmax(1))
    bw = NR.ce_backward(x, w, fw, 0.5)
    assert torch.allclose(bw['dx'], xx.grad, atol=1e-14) and torch.allclose(bw['dW'], ww.grad, atol=1e-13)


def test_first_argmax_is_torch_max_rule():
    nan, inf = float('nan'), float('inf')
    z = torch.tensor([[1., nan, 3., nan], [-inf] * 4, [nan] * 4, [2., 5., 5., 1.], [-inf, -inf, 1., 1.]])
    assert torch.equal(NR.first_argmax(z), z.max(1)[1])
    assert NR.first_argmax(z).tolist() == [1, 0, 0, 1, 2]


# ---------------------------------------------------------------------------------------------------------------- plans
def test_launch_plans():
    assert [NR.bn_row_blocks(n) for n in (2, 512, 513, 524288, 524289, 2 ** 20 + 3)] == [1, 1, 2, 1024, 1024, 1024]
    assert NR.bn_block_rows(524289) == 513 and NR.bn_block_rows(524288) == 512
    assert NR.bn_depth(2) == 1 + 32 + 1 + 8
    assert NR.apply_grid(4097, 34816) == (1, 1088) and NR.apply_grid(4097, 32) == (129, 1)
    assert [NR.ce_splits(n) for n in (63, 1024, 1025, 131071, 131073, 262145)] == [1, 1, 2, 128, 128, 128]
    assert NR.ce_split_rows(262145) == 2049 and NR.ce_row_blocks(262145) == 1024


# ---------------------------------------------------------------------------------------------------------------- bounds
@pytest.mark.parametrize('n,c', [(2, 32), (3, 32), (33, 32), (513, 64), (4097, 32), (20000, 32)])
def test_simulated_statistics_inside_bounds(n, c):
    x, w, b, _ = _rows(n, c, seed=n + c)
    x[:, 1] = 3.25                                                  # constant channel
    st = NR.bn_stats(x, w, b, 1e-5)
    bd = NR.stats_bounds(st)
    sim = _simulated_stats(x, w, b, 1e-5)
    for k in ('mean', 'invstd', 'scale', 'shift'):
        err = (sim[k] - st[k]).abs()
        assert bool((err <= bd[k]).all()), (k, float((err / bd[k]).max()))
        # within about one fp32 half-ulp, not 1e-4
        assert bool((bd[k] <= 1.01 * NR.hu(st[k]) + 1e-6 * NR.hu(st[k]).max()).all()) or k == 'shift'
    rm, rv = torch.rand(c, dtype=torch.float64).float(), (0.5 + torch.rand(c, dtype=torch.float64)).float()
    for momentum in (0.1, None):
        rm_r, rv_r, _, m = NR.bn_running(rm, rv, 4, st, momentum)
        b2 = NR.stats_bounds(st, rm, rv, m)
        rm_k = NR.f32((1.0 - m) * rm.double() + m * sim['mean64'])
        rv_k = NR.f32((1.0 - m) * rv.double() + m * sim['var64'] * n / (n - 1))
        assert bool(((rm_k - rm_r).abs() <= b2['running_mean']).all())
        assert bool(((rv_k - rv_r).abs() <= b2['running_var']).all())
        # negative control: the biased variance in the running buffer
        rv_bad = NR.f32((1.0 - m) * rv.double() + m * sim['var64'])
        assert not bool(((rv_bad - rv_r).abs() <= b2['running_var'])[2:].all())
    # negative control: the momentum-None factor read before the increment (1 / nbt instead of 1 / (nbt + 1))
    rm_r, _, _, m = NR.bn_running(rm, rv, 4, st, None)
    b2 = NR.stats_bounds(st, rm, rv, m)
    rm_bad = NR.f32((1.0 - 0.25) * rm.double() + 0.25 * sim['mean64'])
    assert not bool(((rm_bad - rm_r).abs() <= b2['running_mean']).all())


def test_dropped_last_row_block_breaks_the_bound():
    n, c = 4097, 32                                   # 9 blocks, the last of one row
    x, w, b, _ = _rows(n, c, seed=5, far=10.0)
    st = NR.bn_stats(x, w, b, 1e-5)
    bd = NR.stats_bounds(st)
    rpb = NR.bn_block_rows(n)
    kept = x[:(NR.bn_row_blocks(n) - 1) * rpb]
    sim = _simulated_stats(kept, w, b, 1e-5)
    assert not bool(((sim['mean'] - st['mean']).abs() <= bd['mean']).all())


def _fp32_apply(z, sc, sh, r=None, rsc=None, rsh=None, fma=True):
    """the apply pass in fp32: fmaf(z, sc, sh) (+ r | + fmaf(r, rsc, rsh)), or the unfused multiply-add"""
    def madd(a, s, t):
        return NR.f32(a * s + t) if fma else NR.f32(NR.f32(a * s) + t)
    y = madd(z, sc, sh)
    if r is not None:
        y = NR.f32(y + (r if rsc is None else madd(r, rsc, rsh)))
    return y


@pytest.mark.parametrize('fma', [True, False])
def test_simulated_apply_inside_bound_and_wrong_scale_outside(fma):
    n, c = 2000, 64
    x, w, b, g = _rows(n, c, seed=9)
    r, w2, b2, _ = _rows(n, c, seed=10)
    st, rst = NR.bn_stats(x, w, b, 1e-5), NR.bn_stats(r, w2, b2, 1e-5)
    k, rk = _simulated_stats(x, w, b, 1e-5), _simulated_stats(r, w2, b2, 1e-5)
    for form in ('none', 'identity', 'normalised'):
        for relu in (True, False):
            y_ref, tol = NR.bn_apply(x, st, None if form == 'none' else r, rst if form == 'normalised' else None, relu)
            y = _fp32_apply(x, k['scale'], k['shift'], None if form == 'none' else r,
                            rk['scale'] if form == 'normalised' else None, rk['shift'] if form == 'normalised' else None, fma)
            y = R.split_decode(R.split_of(torch.relu(y) if relu else y), c)
            assert bool(((y - y_ref).abs() <= tol).all()), (form, relu, float(((y - y_ref).abs() / tol).max()))
    # negative control: the downsample residual normalised with the block's own scale / shift
    y_ref, tol = NR.bn_apply(x, st, r, rst, True)
    y = torch.relu(_fp32_apply(x, k['scale'], k['shift'], r, k['scale'], k['shift'], fma))
    assert not bool(((y - y_ref).abs() <= tol).all())
    # negative control: the residual form swapped (identity instead of normalised)
    y = torch.relu(_fp32_apply(x, k['scale'], k['shift'], r, None, None, fma))
    assert not bool(((y - y_ref).abs() <= tol).all())


def test_backward_bounds_and_controls():
    n, c = 3000, 64
    x, w, b, g = _rows(n, c, seed=11, far=100.0)
    st = NR.bn_stats(x, w, b, 1e-5)
    mean32, inv32 = NR.f32(st['mean']), NR.f32(st['invstd'])
    y = torch.relu(x * st['scale'] + st['shift'])
    y[::50, 3] = 0.0                                            # exact zeros: masked by y <= 0
    gin = R.binade_rows(n, c, spread=6, generator=g).double()
    bw = NR.bn_backward(y, gin, x, mean32, inv32, w)
    rb = NR.reduce_bounds(bw)
    # the kernel's order in fp64, then fp32
    xh = (x - mean32) * inv32
    gp = torch.where(y <= 0, torch.zeros_like(gin), gin)
    t1 = torch.zeros(c, dtype=torch.float64)
    t2 = torch.zeros(c, dtype=torch.float64)
    for i in range(n - 1, -1, -1):
        t1 += gp[i]
        t2 += gp[i] * xh[i]
    assert bool(((NR.f32(t1) - bw['t1']).abs() <= rb['dbias']).all())
    assert bool(((NR.f32(t2) - bw['t2']).abs() <= rb['dweight']).all())
    # negative control: the ReLU mask taken as y >= 0 (passes the rows the ReLU clamped to 0)
    bad = NR.bn_backward(None, torch.where(y >= 0, gin, torch.zeros_like(gin)), x, mean32, inv32, w)
    assert not bool(((NR.f32(bad['t1']) - bw['t1']).abs() <= rb['dbias']).all())
    # accumulate: one rounding of prev + t passes, the double rounding prev + fp32(t) does not (on some channel)
    prev = R.binade_rows(1, 4096, spread=2, generator=g)[0].double()
    t = torch.randn(4096, generator=g, dtype=torch.float64) * prev.abs() * 3
    bw_acc = dict(t1=t, t2=t, A1=t.abs(), A2=t.abs(), n=n)
    rb2 = NR.reduce_bounds(bw_acc, prev, prev)
    once = NR.f32(prev + t)
    twice = NR.f32(prev + NR.f32(t))
    assert bool(((once - rb2['db_ref']).abs() <= rb2['dbias']).all())
    assert not bool(((twice - rb2['db_ref']).abs() <= rb2['dbias']).all())
    # dz in fp32 within its bound
    sums = NR.f32(torch.cat([t1, t2]))
    dz_ref, tol = NR.bn_dz(bw, sums)
    a = NR.f32(w.double() * inv32)
    bb, k2 = NR.f32(sums[:c] * NR.f32(torch.tensor(1.0 / n))), NR.f32(sums[c:] * NR.f32(torch.tensor(1.0 / n)))
    xh32 = NR.f32(NR.f32(x - mean32) * inv32)
    dz = NR.f32(a * NR.f32(NR.f32(gp - bb) - xh32 * k2))
    dz = R.split_decode(R.split_of(dz), c)
    assert bool(((dz - dz_ref).abs() <= tol).all()), float(((dz - dz_ref).abs() / tol).max())


def test_ce_dw_bound_holds_for_a_split_order():
    g = torch.Generator().manual_seed(4)
    n, cin, c = 3000, 32, 21
    x = R.binade_rows(n, cin, spread=3, generator=g).double()
    w = torch.randn(cin, c, generator=g) / 6
    perm = torch.randperm(n, generator=g).to(torch.int32)
    lab = torch.randint(0, c, (n,), generator=g)
    fw = NR.ce_forward(x, w, perm, lab, -100)
    bw = NR.ce_backward(x, w, fw, 1.0)
    d32 = NR.f32(bw['d'])
    rps = NR.ce_split_rows(n)
    dW = torch.zeros(cin, c, dtype=torch.float64)
    for s0 in range(0, n, rps):
        acc = torch.zeros(cin, c, dtype=torch.float64)
        for r in range(s0, min(n, s0 + rps)):
            acc = NR.f32(acc + x[r][:, None] * d32[r][None, :])
        dW += acc
    bound = NR.ce_dw_bound(x, bw, n)
    assert bool(((NR.f32(dW) - bw['dW']).abs() <= bound).all())
    # negative control: the split's last row dropped
    dW_bad = dW - x[rps - 1][:, None] * d32[rps - 1][None, :]
    assert not bool(((NR.f32(dW_bad) - bw['dW']).abs() <= bound).all())


# ---------------------------------------------------------------------------------------------------------------- probes
@pytest.mark.parametrize('n', [2, 4, 8, 32, 1024, 2 ** 15])
def test_probe_rows_are_exact_by_construction(n):
    g = torch.Generator().manual_seed(n)
    c = 32
    x, mu, sigma = NR.probe_stats_rows(n, c, generator=g)
    xd = x.double()
    assert torch.equal(xd, x.double().float().double())
    assert torch.equal(R.split_decode(R.split_of(x), c), xd)             # split-exact
    assert torch.equal(xd.mean(0), mu)
    assert torch.equal(((xd - mu) ** 2).mean(0), sigma ** 2)
    assert bool((torch.log2(sigma) == torch.round(torch.log2(sigma))).all())
    if n >= 8:
        far = (xd[0] - mu).abs() / sigma
        assert float(far.max()) >= (n / 4) ** 0.5                         # the pivot row far from the mean somewhere
    w, b = NR.probe_affine(c, generator=g)
    sc = w.double() / sigma
    sh = b.double() - mu * sc
    assert NR.exact_units(sh, 2.0 ** -12) and NR.exact_units(sc, 2.0 ** -12)
    st = NR.bn_stats(xd, w, b, 0.0)
    d = NR.bn_depth(n)
    assert R.exact_budget_bits(st['S2'], 2.0 ** -8) + d.bit_length() < 53
    rm, rv = torch.zeros(c), torch.ones(c)
    erm, erv, tracked = NR.exact_running(rm, rv, 0, mu, sigma, n, None)
    assert tracked == 1 and torch.equal(erm, mu.float()) and torch.equal(erv.double(), (sigma ** 2 * n / (n - 1)).float().double())
