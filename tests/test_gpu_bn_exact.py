"""The six train-mode BatchNorm entry points (csrc/bn_train.cu) and the cross-entropy head (csrc/ce_head.cu) through the C ABI,
element by element against the fp64 references and bounds of tests/norm_ref.py:

* bounds on random operands spanning many binades (means up to 10^3 sigma, a zero-weight channel, a constant channel,
  negative weights) at row counts on both sides of every launch-plan edge (32 row slots, 512-row blocks, the 1024-block cap
  from 524,289 rows on) and channel counts down to one apply block column (34,816);
* bit-exact probes (dyadic values, n a power of two, var a power of four, eps = 0) for every output of all six BatchNorm entry
  points, accumulate modes and ``num_batches_tracked`` included, and for the CE head's argmax with ties planted across the
  32-class chunk edges;
* non-finite inputs follow torch: NaN / inf channels give fp64 ``F.batch_norm(training=True)``'s NaN / inf pattern, ReLU passes
  NaN, the backward of a NaN channel is NaN where torch's is, and a row with a NaN logit has NaN lse / loss and pred = the
  first NaN column (torch's ``max(1)[1]``).

Every output lands in a NaN-filled (or -1-filled) buffer, so a row or channel the kernel never writes fails."""
import pytest
import torch
import torch.nn.functional as F

from openscene_b200 import _cabi as C
from tests import norm_ref as NR
from tests import replay_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAN = float('nan')


def _split(v):
    return R.split_of(v.float()).to(DEV)


def _dec(rows, c):
    return R.split_decode(rows, c)


def _nan(*shape):
    return torch.full(shape, NAN, device=DEV)


def _split_nf(v):
    """split rows that hold +-inf as (inf, 0): the documented split of inf is (inf, bf16(inf - inf) = NaN), which reads back as
    NaN, so an inf input row is written this way"""
    v = v.float()
    hi = v.bfloat16()
    lo = torch.where(torch.isfinite(v), v - hi.float(), torch.zeros_like(v)).bfloat16()
    return R.split_encode(hi, lo).to(DEV)


def _nan_rows(n, c):
    return _split(torch.full((n, c), NAN, device=DEV))


class Stats:
    """one osb_bn_batch_stats(_save) launch with its buffers"""

    def __init__(self, c, w, b, rm, rv, nbt):
        self.c = c
        self.w, self.b = w.to(DEV).float().contiguous(), b.to(DEV).float().contiguous()
        self.rm, self.rv = rm.to(DEV).float().clone(), rv.to(DEV).float().clone()
        self.nbt = torch.full((1,), int(nbt), dtype=torch.int64, device=DEV)
        self.rm0, self.rv0, self.nbt0 = self.rm.clone(), self.rv.clone(), int(nbt)
        self.scale, self.shift, self.mean, self.invstd = _nan(c), _nan(c), _nan(c), _nan(c)

    def run(self, rows, n, eps, momentum, save=True):
        c = self.c
        ws_b = C.lib().osb_bn_stats_workspace_bytes(n, c)
        assert ws_b > 0
        ws = torch.full((ws_b,), 0xFF, dtype=torch.uint8, device=DEV)       # NaN in every fp64 partial slot
        mom = -1.0 if momentum is None else momentum
        common = (C.ptr(rows), n, c, C.ptr(self.w), C.ptr(self.b), eps, mom, C.ptr(self.rm), C.ptr(self.rv), C.ptr(self.nbt),
                  C.ptr(self.scale), C.ptr(self.shift))
        if save:
            C.call('osb_bn_batch_stats_save', *common, C.ptr(self.mean), C.ptr(self.invstd), C.ptr(ws), ws_b, C.stream_ptr())
        else:
            C.call('osb_bn_batch_stats', *common, C.ptr(ws), ws_b, C.stream_ptr())
        torch.cuda.synchronize()

    def reset(self):
        self.rm.copy_(self.rm0)
        self.rv.copy_(self.rv0)
        self.nbt.fill_(self.nbt0)


def _apply(rows, n, c, st, res=None, res_st=None, relu=1, inplace=False):
    args = (n, c, C.ptr(st.scale), C.ptr(st.shift), C.ptr(res), C.ptr(res_st.scale) if res_st else None,
            C.ptr(res_st.shift) if res_st else None, relu, C.stream_ptr())
    if inplace:
        out = rows.clone()
        C.call('osb_bn_apply_split', C.ptr(out), *args)
    else:
        out = _nan_rows(n, c)
        C.call('osb_bn_apply_split_out', C.ptr(rows), C.ptr(out), *args)
    torch.cuda.synchronize()
    return out


def _backward(y_rows, g_rows, z_rows, n, c, st, acc=0, gp_mode=1, dw=None, db=None, gp=None):
    ws_b = C.lib().osb_bn_stats_workspace_bytes(n, c)
    ws = torch.full((ws_b,), 0xFF, dtype=torch.uint8, device=DEV)
    sums = _nan(2 * c)
    dw = _nan(c) if dw is None else dw
    db = _nan(c) if db is None else db
    C.call('osb_bn_backward_reduce', C.ptr(y_rows), C.ptr(g_rows), C.ptr(z_rows), n, c, C.ptr(st.mean), C.ptr(st.invstd),
           C.ptr(sums), C.ptr(dw), C.ptr(db), acc, C.ptr(ws), ws_b, C.stream_ptr())
    dz = _nan_rows(n, c)
    if gp_mode == 0:
        gp = None
    elif gp_mode == 1:
        gp = _nan_rows(n, c)
    C.call('osb_bn_backward_apply', C.ptr(y_rows), C.ptr(g_rows), C.ptr(z_rows), n, c, C.ptr(st.mean), C.ptr(st.invstd),
           C.ptr(st.w), C.ptr(sums), C.ptr(dz), C.ptr(gp), 1 if gp_mode == 2 else 0, C.stream_ptr())
    torch.cuda.synchronize()
    return sums, dw, db, dz, gp


def _within(name, got, ref, bound, worst):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    ok = err <= bound
    assert bool(ok.all()), (name, int((~ok).sum()), float((err / bound.clamp(min=1e-300))[~ok].max()))
    frac = float((err / bound.clamp(min=1e-300)).max()) if err.numel() else 0.0
    worst[name] = max(worst.get(name, 0.0), frac)


# ---------------------------------------------------------------------------------------------------------------- bounds
def _random_case(n, c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sigma = torch.exp(8 * torch.rand(c, device=DEV, generator=g) - 4)              # e^-4 .. e^4
    mean = sigma * (2000 * torch.rand(c, device=DEV, generator=g) - 1000)
    x = mean + sigma * R.binade_rows(n, c, spread=3, generator=g, device=DEV)
    x[:, c - 1] = 3.25                                                               # a constant channel (var 0)
    w = (0.5 + torch.rand(c, device=DEV, generator=g)) * torch.where(torch.rand(c, device=DEV, generator=g) < 0.3, -1.0, 1.0)
    w[0] = 0.0
    b = torch.rand(c, device=DEV, generator=g) - 0.5
    rm, rv = torch.rand(c, device=DEV, generator=g) - 0.5, 0.5 + torch.rand(c, device=DEV, generator=g)
    return _split(x), w, b, rm, rv, g


CASES = ([(n, 32) for n in (2, 3, 31, 32, 33, 511, 512, 513, 4095, 4097, 524287, 524288, 524289, 197383, 2 ** 20 + 3)]
         + [(n, 96) for n in (2, 31, 513, 4097, 197383)] + [(n, 256) for n in (3, 512, 524289)]
         + [(n, 512) for n in (33, 4095, 197383)] + [(n, 34816) for n in (2, 3, 33, 513)])


@pytest.mark.parametrize('n,c', CASES)
def test_batchnorm_bounds(n, c):
    worst = {}
    z_rows, w, b, rm, rv, g = _random_case(n, c, seed=n * 31 + c)
    z = _dec(z_rows, c)
    for momentum in (0.1, None):
        st = Stats(c, w, b, rm, rv, nbt=4)
        st.run(z_rows, n, 1e-5, momentum)
        ref = NR.bn_stats(z, w, b, 1e-5)
        rm_ref, rv_ref, tracked, m = NR.bn_running(rm, rv, 4, ref, momentum)
        bd = NR.stats_bounds(ref, rm, rv, m)
        for k in ('mean', 'invstd', 'scale', 'shift'):
            _within(k, getattr(st, k), ref[k], bd[k], worst)
        _within('running_mean', st.rm, rm_ref, bd['running_mean'], worst)
        _within('running_var', st.rv, rv_ref, bd['running_var'], worst)
        assert int(st.nbt) == tracked == 5
        first = [t.clone() for t in (st.scale, st.shift, st.mean, st.invstd, st.rm, st.rv)]
        st.reset()
        st.run(z_rows, n, 1e-5, momentum, save=False)                # the unsaved entry point: same bits, mean untouched
        assert all(torch.equal(a, b_) for a, b_ in zip(first[:2] + first[4:], [st.scale, st.shift, st.rm, st.rv]))
    # apply against the fp64 statistics, every residual form, ReLU on and off, in place and out of place
    r_rows, w2, b2, _, _, _ = _random_case(n, c, seed=n * 31 + c + 1)
    rst = Stats(c, w2, b2, rm, rv, nbt=0)
    rst.run(r_rows, n, 1e-5, 0.1)
    r = _dec(r_rows, c)
    rref = NR.bn_stats(r, w2, b2, 1e-5)
    for form in ('none', 'identity', 'normalised'):
        for relu in (1, 0):
            res = None if form == 'none' else r_rows
            res_st = rst if form == 'normalised' else None
            y_ref, tol = NR.bn_apply(z, ref, None if form == 'none' else r, rref if res_st else None, bool(relu))
            outs = [_apply(z_rows, n, c, st, res, res_st, relu, inplace=ip) for ip in (False, True)]
            assert torch.equal(outs[0], outs[1])
            _within('apply', _dec(outs[0], c), y_ref, tol, worst)
    # backward on the kernel's own forward (its ReLU mask), all three g' modes and accumulate
    y_rows = _apply(z_rows, n, c, st, r_rows, rst, 1)
    g_rows = _split(R.binade_rows(n, c, spread=4, generator=g, device=DEV))
    y, gin = _dec(y_rows, c), _dec(g_rows, c)
    bw = NR.bn_backward(y, gin, z, st.mean, st.invstd, st.w)
    sums, dw, db, dz, gp = _backward(y_rows, g_rows, z_rows, n, c, st)
    rb = NR.reduce_bounds(bw)
    _within('sums', sums, torch.cat([bw['t1'], bw['t2']]), rb['sums'], worst)
    _within('dbias', db, bw['t1'], rb['dbias'], worst)
    _within('dweight', dw, bw['t2'], rb['dweight'], worst)
    dz_ref, dz_tol = NR.bn_dz(bw, sums)
    _within('dz', _dec(dz, c), dz_ref, dz_tol, worst)
    assert torch.equal(_dec(gp, c), bw['gp'])
    # accumulate onto values independent of t (onto fp32(t) itself a double rounding would go unseen: 2 fp32(t) = fp32(2 t))
    prev_dw = dw * torch.randn(c, device=DEV, generator=g)
    prev_db = db * torch.randn(c, device=DEV, generator=g)
    _, dw2, db2, dz2, gp2 = _backward(y_rows, g_rows, z_rows, n, c, st, acc=1, gp_mode=2, dw=prev_dw.clone(),
                                      db=prev_db.clone(), gp=gp)
    rb2 = NR.reduce_bounds(bw, prev_dw, prev_db)
    _within('dbias_acc', db2, rb2['db_ref'], rb2['dbias'], worst)
    _within('dweight_acc', dw2, rb2['dw_ref'], rb2['dweight'], worst)
    gp2_ref = 2 * NR.f32(bw['gp'])
    _within('gp_acc', _dec(gp2, c), gp2_ref, NR.hu(gp2_ref) + R.OUT_SPLIT * gp2_ref.abs(), worst)
    assert torch.equal(dz2, dz)
    s0, _, _, dz0, _ = _backward(None, g_rows, z_rows, n, c, st, gp_mode=0)             # no ReLU: no mask, no g'
    bw0 = NR.bn_backward(None, gin, z, st.mean, st.invstd, st.w)
    _within('sums', s0, torch.cat([bw0['t1'], bw0['t2']]), NR.reduce_bounds(bw0)['sums'], worst)
    dz0_ref, dz0_tol = NR.bn_dz(bw0, s0)
    _within('dz', _dec(dz0, c), dz0_ref, dz0_tol, worst)
    print('WORST fraction of the bound', n, c, {k: round(v, 3) for k, v in worst.items()})


# ---------------------------------------------------------------------------------------------------------------- exact
PROBES = [(2, 32), (4, 32), (32, 96), (512, 32), (1024, 256), (2 ** 19, 32), (2 ** 20, 32), (4096, 512)]


@pytest.mark.parametrize('n,c', PROBES)
def test_batchnorm_exact_probes(n, c):
    g = torch.Generator().manual_seed(n + c)
    small = n <= 4096
    x, mu, sigma = NR.probe_stats_rows(n, c, generator=g, far_pivot=None if not small else torch.zeros(c, dtype=torch.bool))
    if small:                                   # the dz / g' probe needs xh in {0, +-1} and a narrow sigma range
        x = (mu + (x.double() - mu) / sigma).float()
        sigma = torch.ones(c, dtype=torch.float64)
    w, b = NR.probe_affine(c, generator=g)
    rm = torch.randint(-64, 65, (c,), generator=g).float() * 2.0 ** -6
    rv = torch.randint(1, 65, (c,), generator=g).float() * 2.0 ** -5
    z_rows = _split(x)
    z = _dec(z_rows, c)
    assert torch.equal(z.cpu(), x.double())                      # the probe values are split-exact
    for momentum, nbt in ((0.125, 6), (None, 3)):
        st = Stats(c, w, b, rm, rv, nbt)
        st.run(z_rows, n, 0.0, momentum)
        inv = 1.0 / sigma
        sc = w.double() * inv
        sh = b.double() - mu * sc
        for name, got, exact in (('mean', st.mean, mu), ('invstd', st.invstd, inv), ('scale', st.scale, sc), ('shift', st.shift, sh)):
            assert NR.exact_units(exact, 2.0 ** -12), name
            assert torch.equal(got.cpu(), exact.float()), name
        erm, erv, tracked = NR.exact_running(rm, rv, nbt, mu, sigma, n, momentum)
        assert torch.equal(st.rm.cpu(), erm) and torch.equal(st.rv.cpu(), erv)
        assert int(st.nbt) == tracked
    # apply: y = z scale + shift + r exact in fp32, stored as split(fp32 y)
    r = NR.probe_grid_values((n, c), -4, 2, generator=g)
    r_rows = _split(r)
    rst = Stats(c, torch.full((c,), 0.5), torch.full((c,), 0.25), rm, rv, 0)
    rst.run(z_rows, n, 0.0, 0.5)
    rsc, rsh = 0.5 / sigma, 0.25 - mu * 0.5 / sigma
    for form in ('none', 'identity', 'normalised'):
        for relu in (1, 0):
            t = x.double() * sc + sh
            rr = 0.0 if form == 'none' else (r.double() if form == 'identity' else x.double() * rsc + rsh)
            pre = t + rr
            assert R.exact_budget_bits(t.abs() + (rr.abs() if form != 'none' else 0) + pre.abs(), 2.0 ** -12) < 24
            ex = torch.relu(pre) if relu else pre
            res = None if form == 'none' else (r_rows if form == 'identity' else z_rows.clone())
            out = _apply(z_rows, n, c, st, res, rst if form == 'normalised' else None, relu)
            assert torch.equal(out.cpu(), R.split_of(ex.float())), (form, relu)
    # backward reduce: every sum exact in fp64, one fp32 rounding; accumulate: one rounding of prev + t
    y_rows = _apply(z_rows, n, c, st, r_rows, None, 1)
    # large n: gradients on a finer grid, so the fp64 sums are exact but not fp32-exact and the accumulate's single rounding
    # of prev + t is told apart from a double rounding prev + fp32(t)
    g_lo = -4 if small else -20
    gin = NR.probe_grid_values((n, c), g_lo, 0, generator=g)
    g_rows = _split(gin)
    y = _dec(y_rows, c).cpu()
    bw = NR.bn_backward(y, gin.double(), x.double(), mu.float(), inv.float(), w)
    assert R.exact_budget_bits(bw['A1'] + bw['A2'], 2.0 ** g_lo) < 53
    if not small:
        assert not bool((NR.f32(bw['t1']) == bw['t1']).all())           # some sum is not fp32-exact
    t1, t2 = NR.f32(bw['t1']), NR.f32(bw['t2'])
    sums, dw, db, dz, gp = _backward(y_rows, g_rows, z_rows, n, c, st)
    assert torch.equal(sums.cpu().double(), torch.cat([t1, t2]))
    assert torch.equal(db.cpu().double(), t1) and torch.equal(dw.cpu().double(), t2)
    assert torch.equal(_dec(gp, c).cpu(), bw['gp'])
    prev_w = NR.probe_grid_values((c,), -20, 3, generator=g)
    prev_b = NR.probe_grid_values((c,), -20, 3, generator=g)
    _, dw2, db2, _, gp2 = _backward(y_rows, g_rows, z_rows, n, c, st, acc=1, gp_mode=2, dw=prev_w.to(DEV).clone(),
                                    db=prev_b.to(DEV).clone(), gp=gp)
    assert torch.equal(db2.cpu(), (prev_b.double() + bw['t1']).float())
    assert torch.equal(dw2.cpu(), (prev_w.double() + bw['t2']).float())
    assert torch.equal(_dec(gp2, c).cpu(), 2 * bw['gp'])
    if small:
        # dz = a (g' - b - x^ k2): every fp32 step exact while the budget holds
        a = w.double() * inv
        bb, k2 = t1 / n, t2 / n
        inner = bw['gp'] - bb - bw['xh'] * k2
        dz_ex = a * inner
        grid = 2.0 ** -4 / n * 2.0 ** -2
        mags = torch.stack([bw['gp'].abs().max(0).values, bb.abs(), (bw['xh'] * k2).abs().max(0).values,
                            inner.abs().max(0).values]).max(0).values * a.abs().clamp(min=1)
        assert R.exact_budget_bits(mags, grid) < 24
        assert torch.equal(dz.cpu(), R.split_of(dz_ex.float()))


# ---------------------------------------------------------------------------------------------------------------- non-finite
def test_batchnorm_non_finite_follows_torch():
    n, c = 1000, 32
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(n, c, generator=gen) * 2 + 1
    x[5, 1] = NAN
    x[3, 2] = float('inf')
    x[7, 3] = -float('inf')
    x[9, 4], x[11, 4] = float('inf'), -float('inf')
    x[2, 5], x[4, 5] = NAN, float('inf')
    x[:, 6] = NAN
    w = torch.rand(c, generator=gen) + 0.5
    w[1] = 0.0                                            # a zero weight does not hide a NaN channel
    b = torch.rand(c, generator=gen) - 0.5
    rm, rv = torch.zeros(c), torch.ones(c)
    z_rows = _split_nf(x)
    st = Stats(c, w, b, rm, rv, 0)
    st.run(z_rows, n, 1e-5, 0.1)
    xd = _dec(z_rows, c).cpu().requires_grad_()
    assert bool(torch.isinf(xd[3, 2])) and bool(torch.isnan(xd[5, 1]))
    rm64, rv64 = rm.double(), rv.double()
    w64, b64 = w.double().requires_grad_(), b.double().requires_grad_()
    _, smean, sinv = torch.ops.aten.native_batch_norm(xd.detach(), w64.detach(), b64.detach(), None, None, True, 0.1, 1e-5)
    t = F.batch_norm(xd, rm64, rv64, w64, b64, training=True, momentum=0.1, eps=1e-5)

    def pattern(v):
        v = v.double().cpu()
        return torch.where(torch.isnan(v), 2, torch.where(torch.isinf(v), torch.sign(v).long() * 3, 0))
    ref_sc = w.double() * sinv
    for name, got, ref in (('mean', st.mean, smean), ('invstd', st.invstd, sinv), ('scale', st.scale, ref_sc),
                           ('shift', st.shift, b.double() - smean * ref_sc), ('running_mean', st.rm, rm64),
                           ('running_var', st.rv, rv64)):
        assert torch.equal(pattern(got), pattern(ref)), (name, got[:8], ref[:8])
    for relu in (1, 0):
        y = _dec(_apply(z_rows, n, c, st, relu=relu), c).cpu()
        y_ref = torch.relu(t) if relu else t
        assert torch.equal(pattern(y), pattern(y_ref.detach())), relu
    # the backward of relu(BN(z)): NaN channels give torch's NaN pattern (threshold_backward passes a NaN output's gradient)
    y_rows = _apply(z_rows, n, c, st, relu=1)
    gin = torch.randn(n, c, generator=gen)
    g_rows = _split(gin)
    torch.relu(t).backward(_dec(g_rows, c).cpu())
    _, dw, db, dz, _ = _backward(y_rows, g_rows, z_rows, n, c, st)
    assert torch.equal(pattern(dw), pattern(w64.grad)) and torch.equal(pattern(db), pattern(b64.grad))
    assert bool(torch.isnan(dw[[1, 2, 3, 4, 5, 6]]).all()) and bool(torch.isfinite(db).all())
    # dbias is the sum of g where the kernel's own output is not <= 0 (NaN rows included)
    yk, gk = _dec(y_rows, c).cpu(), _dec(g_rows, c).cpu()
    db_ref = torch.where(yk <= 0, torch.zeros_like(gk), gk).sum(0)
    assert torch.allclose(db.double().cpu(), db_ref, rtol=1e-6, atol=1e-6)
    assert bool(torch.isnan(_dec(dz, c)[:, 1:7]).all()) and bool(torch.isfinite(_dec(dz, c)[:, 7:]).all())
    # a non-finite value in row 0 (the shift pivot of the fp64 sums): torch's mean is +-inf, the kernel's NaN; everything
    # that depends on the mean is NaN in both
    x0 = torch.randn(64, 32, generator=gen)
    x0[0, 0] = float('inf')
    st0 = Stats(32, torch.ones(32), torch.zeros(32), torch.zeros(32), torch.ones(32), 0)
    st0.run(_split_nf(x0), 64, 1e-5, 0.1)
    assert bool(torch.isnan(st0.mean[0])) and bool(torch.isnan(st0.shift[0])) and bool(torch.isnan(st0.rv[0]))
    assert bool(torch.isfinite(st0.mean[1:]).all())


# ---------------------------------------------------------------------------------------------------------------- CE head
def _ce_run(xs, n, cin, w, c, perm, lab, ignore, g=1.0):
    ws_b = C.lib().osb_ce_head_workspace_bytes(n, cin, c)
    ws = torch.full((ws_b,), 0xFF, dtype=torch.uint8, device=DEV)
    lse = _nan(n)
    pred = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    loss = _nan(1)
    nv = torch.full((1,), -1, dtype=torch.int64, device=DEV)
    i64 = 1 if lab.dtype == torch.int64 else 0
    C.call('osb_ce_head_fwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(perm), C.ptr(lab), i64, ignore, C.ptr(lse), C.ptr(pred),
           C.ptr(loss), C.ptr(nv), C.ptr(ws), ws_b, C.stream_ptr())
    gt = torch.full((1,), g, device=DEV)
    dx = _nan_rows(n, cin)
    dw = _nan(cin, c)
    C.call('osb_ce_head_bwd', C.ptr(xs), n, cin, C.ptr(w), c, C.ptr(perm), C.ptr(lab), i64, ignore, C.ptr(lse), C.ptr(gt),
           C.ptr(nv), C.ptr(dx), C.ptr(dw), C.ptr(ws), ws_b, C.stream_ptr())
    torch.cuda.synchronize()
    return lse, pred, loss, nv, dx, dw


def _ce_case(n, cin, c, seed, i64=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = R.binade_rows(n, cin, spread=3, generator=g, device=DEV)
    w = torch.randn(cin, c, device=DEV, generator=g) / cin ** 0.5
    perm = torch.randperm(n, device=DEV, generator=g).to(torch.int32)
    lab = torch.randint(0, c, (n,), device=DEV, generator=g)
    lab[torch.rand(n, device=DEV, generator=g) < 0.15] = 255
    return _split(x), w, perm, lab.to(torch.int64 if i64 else torch.int32)


CE_CASES = ([(n, cin, c) for n in (63, 65, 1025) for cin in (32, 384) for c in (1, 31, 32, 33, 65, 159, 160)]
            + [(n, cin, c) for n in (63, 64, 65, 1024, 1025, 131071, 131073, 262145) for cin, c in ((32, 33), (384, 160), (96, 20))])


@pytest.mark.parametrize('n,cin,c', CE_CASES)
def test_ce_head_bounds(n, cin, c):
    worst = {}
    xs, w, perm, lab = _ce_case(n, cin, c, seed=n + 7 * cin + c, i64=(n % 2 == 1))
    lse, pred, loss, nv, dx, dw = _ce_run(xs, n, cin, w, c, perm, lab, 255, g=0.75)
    x = _dec(xs, cin)
    fw = NR.ce_forward(x, w, perm, lab, 255)
    assert int(nv) == fw['n_valid']
    assert torch.allclose(lse.double(), fw['lse'], rtol=2 ** -20, atol=2 ** -20 * float(fw['lse'].abs().max()))
    assert abs(float(loss) - float(fw['loss'])) <= 2 ** -20 * abs(float(fw['loss']))
    z = fw['z']
    top2 = z.topk(min(2, c), 1).values
    gap = top2[:, 0] - top2[:, 1] if c > 1 else torch.full((n,), float('inf'), dtype=torch.float64, device=DEV)
    sure = gap > 2 ** -18 * z.abs().max(1).values
    assert bool((pred >= 0).all()) and torch.equal(pred[perm.long()][sure], fw['pred_int'][sure])
    bw = NR.ce_backward(x, w, fw, 0.75)
    _within('ce_dx', _dec(dx, cin), bw['dx'], NR.ce_dx_bound(w, bw) + 1e-300, worst)
    _within('ce_dW', dw, bw['dW'], NR.ce_dw_bound(x, bw, n) + 1e-300, worst)
    again = _ce_run(xs, n, cin, w, c, perm, lab, 255, g=0.75)
    assert all(torch.equal(a, b) for a, b in zip((lse, pred, loss, nv, dx, dw), again))
    print('WORST fraction of the bound', n, cin, c, {k: round(v, 3) for k, v in worst.items()})


@pytest.mark.parametrize('n', [65, 1025, 131073])
@pytest.mark.parametrize('cin', [32, 384])
def test_ce_head_exact_pred_with_ties(n, cin):
    """dyadic x and W: every logit is exact in fp32, so pred must be the first maximum bit for bit; ties planted across the
    32-class chunk edges (31|32, 127|128) and with the last class (63|159)"""
    c = 160
    g = torch.Generator().manual_seed(n + cin)
    x = NR.probe_grid_values((n, cin), -3, 0, generator=g)
    w = NR.probe_grid_values((cin, c), -4, -1, generator=g)
    for a, b in ((31, 32), (127, 128), (63, 159)):
        w[:, b] = w[:, a]
    # make the tied pairs the maximum on many rows: channel 0 of a row lifts the pair 31|32 (x = 2) or 127|128 (x = -2)
    x[:, 0] = torch.tensor([2.0, -2.0, 0.0])[torch.randint(3, (n,), generator=g)]
    w[0, :] = 0.0
    w[0, 31] = w[0, 32] = 32.0
    w[0, 127] = w[0, 128] = -32.0
    # channel 1 lifts the pair 63|159 (the last class, in the last chunk) on the rows where x[:, 1] = 2 and x[:, 0] = 0
    x[:, 1] = torch.where(x[:, 0] == 0, torch.tensor(2.0), torch.tensor(0.0))
    w[1, :] = 0.0
    w[1, 63] = w[1, 159] = 32.0
    z = x.double() @ w.double()
    assert R.exact_budget_bits(x.double().abs() @ w.double().abs(), 2.0 ** -7) < 24
    perm = torch.randperm(n, generator=g).to(torch.int32)
    lab = torch.randint(0, c, (n,), generator=g)
    xs = _split(x)
    lse, pred, *_ = _ce_run(xs, n, cin, w.to(DEV), c, perm.to(DEV), lab.to(DEV), -100)
    ref = NR.first_argmax(z)
    got = pred.cpu()[perm.long()]
    assert torch.equal(got, ref)
    for a, b in ((31, 32), (127, 128), (63, 159)):
        assert bool((got == a).any()) and not bool((got == b).any())


def test_ce_head_nan_logits_follow_torch():
    """rows with x NaN: every logit NaN (pred 0); W[5, 37] = W[5, 90] = inf on rows with x[:, 5] = 0: NaN at 37 and 90 only,
    so pred is 37, the first NaN; lse NaN on those rows and the loss NaN, n_valid unchanged"""
    n, cin, c = 300, 32, 100
    g = torch.Generator().manual_seed(1)
    x = NR.probe_grid_values((n, cin), -3, 0, generator=g)
    x[:, 5] = 0.0
    x[10:20, 3] = NAN
    w = NR.probe_grid_values((cin, c), -4, -1, generator=g)
    w[5, 37] = w[5, 90] = float('inf')
    perm = torch.randperm(n, generator=g).to(torch.int32)
    lab = torch.randint(0, c, (n,), generator=g)
    lab[::2] = 255
    lse, pred, loss, nv, *_ = _ce_run(_split(x), n, cin, w.to(DEV), c, perm.to(DEV), lab.to(DEV), 255)
    z = x.double() @ w.double()
    assert bool(torch.isnan(z).any(1).all())
    got = pred.cpu()[perm.long()]
    assert torch.equal(got, NR.first_argmax(z))
    assert torch.equal(got, z.float().max(1)[1])                   # torch's own rule on the same logits
    assert bool((got[10:20] == 0).all()) and bool((got[20:] == 37).all())
    assert bool(torch.isnan(lse).all()) and bool(torch.isnan(loss).all())
    assert int(nv) == int((lab != 255).sum())
