"""Every BatchNorm and cross-entropy launch of the engines replayed in fp64 on the operands it read, and the wiring checked.

The end-to-end yardsticks (tests/test_gpu_bn_batch_stats.py, tests/test_gpu_engine_train*.py) cannot see an error below about
1e-3 .. 1e-2 in one layer, and tests/test_gpu_bn_exact.py calls the kernels in isolation.  Here the library the engine sees is
a wrapper (as in tests/test_gpu_launch_replay.py): it records every convolution launch's output (pointer, rows, channels) and
passes it through, and around every BatchNorm / CE launch it synchronises, snapshots the operands, launches the real entry point,
snapshots what it wrote and compares that with tests/norm_ref.py element by element, within its per-element bound.  Wiring:

* every BatchNorm1d has exactly one statistics launch per forward (found through its weight / bias / running-buffer
  pointers), and it reads the rows a convolution just wrote, with that convolution's rows and channels;
* apply reads that launch's scale / shift; its residual is either rows an earlier apply wrote (the block input) or the raw
  rows of a downsample convolution with the downsample BatchNorm's own scale / shift;
* in training, reduce and apply read this step's saved mean / invstd and the forward's raw rows, the mask is the BatchNorm's
  own apply output -- for a downsample BatchNorm the output of the block it feeds -- an accumulating g' continues a buffer an
  earlier launch wrote, and after backward() the last dweight / dbias of each BatchNorm equal bn.weight.grad / bn.bias.grad
  bit for bit;
* the CE head reads the trunk's last activation, final.kernel and the row permutation the input gather used, and its dW is
  final.kernel.grad;
* the cosine head (``forward_train_cosine``, driven with ``(0.75 * loss).backward()`` so that a dropped upstream gradient
  shows) reads the last apply's output with its rows and width, final.kernel, the caller's targets and, as supervised rows,
  the inverse of the input gather's permutation at the caller's mask rows in caller order; its backward reads the forward's
  rows, weights, row index, targets and state (unchanged since the forward wrote it) and g = 0.75; its dW is
  final.kernel.grad and its dx is the gradient the first BatchNorm backward reduce and apply read.  Both launches are compared
  with ``cos_ref.head`` element by element.

Reference-side negative controls must fail: a swapped residual form, the block's own BatchNorm on the downsample residual, a
dropped mask, and for the cosine head rows taken through the permutation instead of its inverse, targets rolled by one row
and g = 1.  An entry point that is neither handled nor on the pass-through list fails the run."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import collections, sys, torch
sys.path.insert(0, %(root)r)
cfg = sys.argv[1]
from openscene_b200 import engine, synth, _cabi as C
from tests import cos_ref as CR
from tests import norm_ref as NR
from tests import replay_ref as R

dev = torch.device('cuda:0')

PASS = {
    'osb_bn_stats_workspace_bytes', 'osb_ce_head_workspace_bytes', 'osb_cos_head_workspace_bytes', 'osb_f32_to_split', 'osb_split_to_f32',
    'osb_kernel_map_build', 'osb_kernel_map_build_grid', 'osb_kernel_map_transpose', 'osb_hash_build',
    'osb_coordset_build', 'osb_coordset_stride', 'osb_coordset_pyramid', 'osb_coordset_workspace_bytes',
    'osb_occgrid_build', 'osb_occgrid_bytes', 'osb_folded_head_finish', 'osb_conv_wgrad_tc',
    'osb_conv_pack_weights', 'osb_conv_pack_weight_tiles', 'osb_conv_packed_weight_bytes', 'osb_conv_weight_tiles_bytes',
    'osb_conv_tc_workspace_bytes', 'osb_conv_chain_workspace_bytes', 'osb_conv_wgrad_tc_workspace_bytes',
    'osb_conv_desc_bytes', 'osb_conv_chain_grid', 'osb_last_error', 'osb_tuning_set', 'osb_conv_fwd_f32',
}
HANDLED = ('osb_conv_fwd_tc', 'osb_conv_desc_fill', 'osb_conv_chain_launch', 'osb_convtr_fwd_tc', 'osb_conv_stem_fused',
           'osb_conv_stem_fused_grid', 'osb_gather_rows_f32', 'osb_bn_batch_stats', 'osb_bn_batch_stats_save',
           'osb_bn_apply_split', 'osb_bn_apply_split_out', 'osb_bn_backward_reduce', 'osb_bn_backward_apply',
           'osb_ce_head_fwd', 'osb_ce_head_bwd', 'osb_cos_head_fwd', 'osb_cos_head_bwd')


def _i(a):
    return 0 if a is None else (a if isinstance(a, (int, float)) else (a.value or 0))


class _Raw:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (ptr, False), 'version': 3}


def snap(ptr, nbytes):
    return torch.as_tensor(_Raw(ptr, nbytes), device=dev).clone()


def f32(ptr, n):
    return snap(ptr, 4 * n).view(torch.float32)


def rows(ptr, n, c):
    return R.split_decode(snap(ptr, n * 4 * c).view(n, -1), c)


class Harness:
    def __init__(self, model):
        self.real = C.lib()
        self.model = model
        self.bn_of = {}                                   # weight pointer -> BatchNorm name
        for name, m in model.named_modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                self.bn_of[m.weight.data_ptr()] = name
        self.produced = {}                                 # pointer -> (rows, channels) of the latest convolution writing it
        self.descs = {}
        self.stats = []                                    # statistics launches of the current forward, in order
        self.applies = []                                  # apply launches
        self.written = set()                               # every buffer a backward launch wrote
        self.reduce_last = {}                              # BatchNorm name -> (dweight, dbias) of its latest reduce
        self.last_bw = None
        self.counts = collections.Counter()
        self.worst = collections.defaultdict(float)
        self.neg = collections.Counter()
        self.gather_perm = None
        self.ce = {}
        self.cos = {}
        self.cos_caller = None                             # (caller rows of the mask, feat_3d, g) of a cosine step
        self.cos_dx_readers = {}                           # BatchNorm backward entry point -> the dx it must read as g

    def __getattr__(self, name):
        if name in PASS:
            return getattr(self.real, name)
        if name in HANDLED:
            return getattr(self, '_' + name[4:])
        raise AssertionError(f"entry point {name} is neither replayed nor on the pass-through list")

    def call(self, name, *a):
        C.check(getattr(self, name)(*a), name)

    def within(self, op, got, ref, bound):
        err = (got.double() - ref).abs()
        ok = err <= bound
        assert bool(ok.all()), f"{op}: {int((~ok).sum())} elements outside the bound, worst {float((err / bound.clamp(min=1e-300))[~ok].max()):.3g}"
        if err.numel():
            self.worst[op] = max(self.worst[op], float((err / bound.clamp(min=1e-300)).max()))

    def fails(self, got, ref, bound):
        return not bool(((got.double() - ref).abs() <= bound).all())

    # ------------------------------------------------------------ convolutions: record the output, pass through
    def _conv_fwd_tc(self, *args):
        rc = self.real.osb_conv_fwd_tc(*args)
        a = [_i(v) for v in args]
        if not rc and a[15]:
            self.produced[a[15]] = (a[7], a[10])
            self.written.add(a[15])
        return rc

    def _conv_desc_fill(self, *args):
        a = [_i(v) for v in args]
        self.descs[a[0]] = (a[14], a[6], a[9], a[17], a[18])
        return self.real.osb_conv_desc_fill(*args)

    def _conv_chain_launch(self, *args):
        rc = self.real.osb_conv_chain_launch(*args)
        a = [_i(v) for v in args]
        db = self.real.osb_conv_desc_bytes()
        for i in range(a[1]):
            out, n_out, cout, cmap, cmap_cout = self.descs[a[0] + i * db]
            if cmap:
                torch.cuda.synchronize()
                n_out = int((snap(cmap, 8 * n_out * 4).view(torch.int32) >= 0).sum())
                cout = cmap_cout
            if out:
                self.produced[out] = (n_out, cout)
        return rc

    def _convtr_fwd_tc(self, *args):
        rc = self.real.osb_convtr_fwd_tc(*args)
        a = [_i(v) for v in args]
        torch.cuda.synchronize()
        n_f = int((snap(a[3], 8 * a[2] * 4).view(torch.int32) >= 0).sum())
        if a[10]:
            self.produced[a[10]] = (n_f, a[6])
        return rc

    def _stem(self, name, args, grid):
        rc = getattr(self.real, name)(*args)
        a = [_i(v) for v in args]
        cout = a[11] if grid else a[9]
        if a[-3]:
            self.produced[a[-3]] = (a[3], cout)
        return rc

    def _conv_stem_fused(self, *args):
        return self._stem('osb_conv_stem_fused', args, False)

    def _conv_stem_fused_grid(self, *args):
        return self._stem('osb_conv_stem_fused_grid', args, True)

    def _gather_rows_f32(self, *args):
        a = [_i(v) for v in args]
        self.gather_perm = (a[1], a[2])
        return self.real.osb_gather_rows_f32(*args)

    # ------------------------------------------------------------ statistics
    def _stats(self, name, args, save):
        a = [_i(v) for v in args]
        x_a, n, c, w_a, b_a, eps, mom, rm_a, rv_a, nbt_a, sc_a, sh_a = a[:12]
        mean_a, inv_a = (a[12], a[13]) if save else (0, 0)
        torch.cuda.synchronize()
        assert self.produced.get(x_a) == (n, c), f"statistics launch reads rows {self.produced.get(x_a)} no convolution wrote as ({n}, {c})"
        bn = self.bn_of.get(w_a)
        assert bn is not None, "statistics launch with weights of no BatchNorm1d"
        x = rows(x_a, n, c)
        w, b, rm, rv = f32(w_a, c), f32(b_a, c), f32(rm_a, c), f32(rv_a, c)
        nbt = int(snap(nbt_a, 8).view(torch.int64))
        rc = getattr(self.real, name)(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts[name] += 1
        momentum = None if mom < 0 else mom
        st = NR.bn_stats(x, w, b, eps)
        rm_ref, rv_ref, tracked, m = NR.bn_running(rm, rv, nbt, st, momentum)
        bd = NR.stats_bounds(st, rm, rv, m)
        for k, p in (('scale', sc_a), ('shift', sh_a), ('mean', mean_a), ('invstd', inv_a)):
            if p:
                self.within('stats-' + k, f32(p, c), st[k], bd[k])
        self.within('running_mean', f32(rm_a, c), rm_ref, bd['running_mean'])
        self.within('running_var', f32(rv_a, c), rv_ref, bd['running_var'])
        assert int(snap(nbt_a, 8).view(torch.int64)) == tracked
        self.stats.append(dict(bn=bn, x=x_a, n=n, c=c, scale=sc_a, shift=sh_a, mean=mean_a, invstd=inv_a, w=w_a, st=st))
        return 0

    def _bn_batch_stats(self, *args):
        return self._stats('osb_bn_batch_stats', args, False)

    def _bn_batch_stats_save(self, *args):
        return self._stats('osb_bn_batch_stats_save', args, True)

    def stats_of(self, x_a):
        hit = [s for s in self.stats if s['x'] == x_a]
        assert hit, "rows with no statistics launch"
        return hit[-1]

    # ------------------------------------------------------------ apply
    def _apply(self, name, args, out_of_place):
        a = [_i(v) for v in args]
        if out_of_place:
            x_a, y_a, n, c, sc_a, sh_a, r_a, rsc_a, rsh_a, relu = a[:10]
        else:
            x_a, n, c, sc_a, sh_a, r_a, rsc_a, rsh_a, relu = a[:9]
            y_a = x_a
        torch.cuda.synchronize()
        S = self.stats_of(x_a)
        assert (S['scale'], S['shift'], S['n'], S['c']) == (sc_a, sh_a, n, c), \
            f"{S['bn']}: apply does not read its statistics launch's scale / shift"
        x = rows(x_a, n, c)
        res, RS = None, None
        if r_a:
            res = rows(r_a, n, c)
            if rsc_a:
                RS = self.stats_of(r_a)
                assert (RS['scale'], RS['shift']) == (rsc_a, rsh_a), \
                    f"{S['bn']}: the downsample residual is not normalised with its own BatchNorm's scale / shift"
                assert RS['bn'] != S['bn']
            else:
                assert any(A['y'] == r_a for A in self.applies), f"{S['bn']}: identity residual that no apply wrote"
        rc = getattr(self.real, name)(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts[name] += 1
        y = rows(y_a, n, c)
        ref, tol = NR.bn_apply(x, S['st'], res, RS['st'] if RS else None, bool(relu))
        self.within('apply', y, ref, tol)
        if RS is not None and not self.neg['swapped_form']:
            r2, t2 = NR.bn_apply(x, S['st'], res, None, bool(relu))
            assert self.fails(y, r2, t2), "negative control: a swapped residual form passed"
            self.neg['swapped_form'] += 1
        if RS is not None and not self.neg['own_bn_on_downsample']:
            r2, t2 = NR.bn_apply(x, S['st'], res, S['st'], bool(relu))
            assert self.fails(y, r2, t2), "negative control: the block's own BatchNorm on the downsample residual passed"
            self.neg['own_bn_on_downsample'] += 1
        self.applies.append(dict(bn=S['bn'], x=x_a, y=y_a, res=r_a, res_bn=RS['bn'] if RS else None, relu=relu, n=n, c=c))
        return 0

    def _bn_apply_split(self, *args):
        return self._apply('osb_bn_apply_split', args, False)

    def _bn_apply_split_out(self, *args):
        return self._apply('osb_bn_apply_split_out', args, True)

    # ------------------------------------------------------------ backward
    def check_backward_operands(self, y_a, z_a, n, c, mean_a, inv_a):
        S = self.stats_of(z_a)
        assert (S['n'], S['c'], S['mean'], S['invstd']) == (n, c, mean_a, inv_a), \
            f"{S['bn']}: the backward does not read its forward's raw rows / saved mean / invstd"
        own = [A for A in self.applies if A['x'] == z_a]
        if own:
            want = own[-1]['y']
        else:                                              # a downsample BatchNorm: the output of the block it feeds
            fed = [A for A in self.applies if A['res'] == z_a and A['res_bn'] == S['bn']]
            assert fed, f"{S['bn']}: no apply consumed its rows"
            want = fed[-1]['y']
        assert y_a == want, f"{S['bn']}: the backward mask is not the output its rows fed"
        return S

    def _bn_backward_reduce(self, *args):
        a = [_i(v) for v in args]
        y_a, g_a, z_a, n, c, mean_a, inv_a, sums_a, dw_a, db_a, acc = a[:11]
        torch.cuda.synchronize()
        self.cos_gradient_read('osb_bn_backward_reduce', g_a)
        S = self.check_backward_operands(y_a, z_a, n, c, mean_a, inv_a)
        y, g, z = rows(y_a, n, c) if y_a else None, rows(g_a, n, c), rows(z_a, n, c)
        mean, inv, w = f32(mean_a, c), f32(inv_a, c), f32(S['w'], c)
        prev = (f32(dw_a, c), f32(db_a, c)) if acc else (None, None)
        rc = self.real.osb_bn_backward_reduce(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_bn_backward_reduce'] += 1
        bw = NR.bn_backward(y, g, z, mean, inv, w)
        rb = NR.reduce_bounds(bw, *prev)
        sums = f32(sums_a, 2 * c)
        self.within('reduce-sums', sums, torch.cat([bw['t1'], bw['t2']]), rb['sums'])
        dw, db = f32(dw_a, c), f32(db_a, c)
        self.within('dweight', dw, rb['dw_ref'], rb['dweight'])
        self.within('dbias', db, rb['db_ref'], rb['dbias'])
        if y is not None and not self.neg['dropped_mask']:
            bad = NR.bn_backward(None, g, z, mean, inv, w)
            if bool((bad['t1'] != bw['t1']).any()):
                assert self.fails(db, bad['t1'], rb['dbias']), "negative control: a dropped mask passed"
                self.neg['dropped_mask'] += 1
        self.reduce_last[S['bn']] = (dw, db)
        self.last_bw = dict(key=(y_a, g_a, z_a, sums_a), bw=bw)
        return 0

    def _bn_backward_apply(self, *args):
        a = [_i(v) for v in args]
        y_a, g_a, z_a, n, c, mean_a, inv_a, w_a, sums_a, dz_a, gp_a, gp_acc = a[:12]
        torch.cuda.synchronize()
        self.cos_gradient_read('osb_bn_backward_apply', g_a)
        S = self.check_backward_operands(y_a, z_a, n, c, mean_a, inv_a)
        assert w_a == S['w'], f"{S['bn']}: backward apply reads another weight"
        assert self.last_bw and self.last_bw['key'] == (y_a, g_a, z_a, sums_a), f"{S['bn']}: apply without its reduce"
        bw = self.last_bw['bw']
        sums = f32(sums_a, 2 * c)
        prev_gp = None
        if gp_acc:
            assert gp_a in self.written, f"{S['bn']}: an accumulating g' onto a buffer no earlier launch wrote"
            prev_gp = rows(gp_a, n, c)
        rc = self.real.osb_bn_backward_apply(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_bn_backward_apply'] += 1
        dz_ref, tol = NR.bn_dz(bw, sums)
        self.within('dz', rows(dz_a, n, c), dz_ref, tol)
        if gp_a:
            gp = rows(gp_a, n, c)
            if gp_acc:
                ref = prev_gp + bw['gp']
                self.within('gp-accumulate', gp, ref, NR.hu(ref) * 1.0001 + R.OUT_SPLIT * ref.abs())
            else:
                assert torch.equal(gp, bw['gp']), f"{S['bn']}: g' is not the masked gradient"
            self.written.add(gp_a)
        self.written.add(dz_a)
        return 0

    # ------------------------------------------------------------ cross-entropy head
    def _ce_head_fwd(self, *args):
        a = [_i(v) for v in args]
        x_a, n, cin, w_a, c, rm_a, lab_a, i64, ignore, lse_a, pred_a, loss_a, nv_a = a[:13]
        torch.cuda.synchronize()
        assert self.applies and self.applies[-1]['y'] == x_a, "the CE head does not read the trunk's last activation"
        assert self.gather_perm is not None and self.gather_perm == (rm_a, n), "the CE head's row map is not the input permutation"
        x, w = rows(x_a, n, cin), f32(w_a, cin * c).view(cin, c)
        perm = snap(rm_a, 4 * n).view(torch.int32)
        lab = snap(lab_a, (8 if i64 else 4) * n).view(torch.int64 if i64 else torch.int32)
        rc = self.real.osb_ce_head_fwd(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_ce_head_fwd'] += 1
        fw = NR.ce_forward(x, w, perm, lab, ignore)
        lse = f32(lse_a, n).double()
        assert torch.allclose(lse, fw['lse'], rtol=2 ** -20, atol=2 ** -20 * float(fw['lse'].abs().max()))
        assert int(snap(nv_a, 8).view(torch.int64)) == fw['n_valid']
        loss = float(f32(loss_a, 1))
        assert abs(loss - float(fw['loss'])) <= 2 ** -20 * abs(float(fw['loss']))
        z = fw['z']
        top2 = z.topk(min(2, c), 1).values
        sure = (top2[:, 0] - top2[:, 1]) > 2 ** -18 * z.abs().max(1).values
        pred = snap(pred_a, 8 * n).view(torch.int64)
        assert torch.equal(pred[perm.long()][sure], fw['pred_int'][sure])
        self.ce = dict(x=x_a, w=w_a, w_val=w, fw=fw, xv=x)
        return 0

    def _ce_head_bwd(self, *args):
        a = [_i(v) for v in args]
        x_a, n, cin, w_a, c = a[:5]
        g_a, dx_a, dw_a = a[10], a[12], a[13]
        torch.cuda.synchronize()
        assert (x_a, w_a) == (self.ce['x'], self.ce['w']), "the CE backward does not read its forward's rows and weights"
        g = float(f32(g_a, 1))
        rc = self.real.osb_ce_head_bwd(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_ce_head_bwd'] += 1
        bw = NR.ce_backward(self.ce['xv'], self.ce['w_val'], self.ce['fw'], g)
        dw = f32(dw_a, cin * c).view(cin, c)
        self.within('ce-dW', dw, bw['dW'], NR.ce_dw_bound(self.ce['xv'], bw, n) + 1e-300)
        self.within('ce-dx', rows(dx_a, n, cin), bw['dx'], NR.ce_dx_bound(self.ce['w_val'], bw) + 1e-300)
        self.ce['dW'] = dw
        self.written.add(dx_a)
        return 0

    # ------------------------------------------------------------ cosine head
    def cos_within(self, got, ref):
        for k, v in got.items():
            r = CR.ratio(v, *ref[k])
            assert r <= 1, f"cos-{k}: {r:.3g} of the bound"
            self.worst['cos-' + k] = max(self.worst['cos-' + k], r)

    def cos_fails(self, got, ref):
        return any(CR.ratio(v, *ref[k]) > 1 for k, v in got.items())

    def _cos_head_fwd(self, *args):
        a = [_i(v) for v in args]
        x_a, n, cin, w_a, c, rows_a, m, t_a, st_a, loss_a = a[:10]
        torch.cuda.synchronize()
        A = self.applies[-1] if self.applies else None
        assert A is not None and (A['y'], A['n'], A['c']) == (x_a, n, cin), "the cosine head does not read the trunk's last activation"
        assert w_a == self.model.final.kernel.data_ptr() and (cin, c) == tuple(self.model.final.kernel.shape[-2:]), \
            "the cosine head does not read final.kernel"
        caller, feat, _ = self.cos_caller
        assert t_a == feat.data_ptr() and m == feat.shape[0] == caller.numel(), "the cosine head does not read the caller's targets"
        assert self.gather_perm is not None and self.gather_perm[1] == n, "no input gather before the cosine head"
        perm = snap(self.gather_perm[0], 4 * n).view(torch.int32).long()
        inv = torch.empty_like(perm)
        inv[perm] = torch.arange(n, device=dev)
        sel = snap(rows_a, 4 * m).view(torch.int32)
        assert torch.equal(sel.long(), inv[caller]), "the cosine head's rows are not the inverse gather permutation at the caller's rows"
        x, w = rows(x_a, n, cin), f32(w_a, cin * c).view(cin, c)
        t = snap(t_a, 2 * m * c).view(torch.float16).view(m, c).double()
        rc = self.real.osb_cos_head_fwd(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_cos_head_fwd'] += 1
        state = snap(st_a, 24 * m).view(torch.float64).view(m, 3)
        got = dict(state=state, loss=f32(loss_a, 1)[0])
        self.cos_within(got, CR.head(x, w, t, sel, 1.0))
        if not self.neg['cos_rows_through_perm']:
            assert self.cos_fails(got, CR.head(x, w, t, perm[caller], 1.0)), "negative control: rows through perm passed"
            self.neg['cos_rows_through_perm'] += 1
        if not self.neg['cos_targets_rolled']:
            assert self.cos_fails(got, CR.head(x, w, t.roll(1, 0), sel, 1.0)), "negative control: rolled targets passed"
            self.neg['cos_targets_rolled'] += 1
        self.cos = dict(args=(x_a, n, cin, w_a, c, rows_a, m, t_a, st_a), x=x, w=w, t=t, sel=sel, state=state)
        return 0

    def _cos_head_bwd(self, *args):
        a = [_i(v) for v in args]
        x_a, n, cin, w_a, c, rows_a, m, t_a, st_a, g_a, dx_a, dw_a = a[:12]
        torch.cuda.synchronize()
        F = self.cos
        assert F and F['args'] == (x_a, n, cin, w_a, c, rows_a, m, t_a, st_a), \
            "the cosine backward does not read its forward's rows, weights, row index, targets and state"
        assert torch.equal(rows(x_a, n, cin), F['x']) and torch.equal(f32(w_a, cin * c).view(cin, c), F['w']), \
            "the cosine head's rows or weights changed between forward and backward"
        assert torch.equal(snap(rows_a, 4 * m).view(torch.int32), F['sel'])
        assert torch.equal(snap(t_a, 2 * m * c).view(torch.float16).view(m, c).double(), F['t'])
        assert torch.equal(snap(st_a, 24 * m).view(torch.float64).view(m, 3).view(torch.int64), F['state'].view(torch.int64)), \
            "the cosine state changed between forward and backward"
        g = float(f32(g_a, 1))
        assert g == self.cos_caller[2], f"the cosine backward reads g = {g}, not the upstream gradient {self.cos_caller[2]}"
        rc = self.real.osb_cos_head_bwd(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_cos_head_bwd'] += 1
        dx = rows(dx_a, n, cin)
        r = F['sel'].long()
        others = torch.ones(n, dtype=torch.bool, device=dev)
        others[r] = False
        assert bool((dx[others] == 0).all()), "the cosine dx is not 0 on the unsupervised rows"
        dw = f32(dw_a, cin * c).view(cin, c)
        got = dict(dx=dx[r], dW=dw)
        self.cos_within(got, CR.head(F['x'], F['w'], F['t'], F['sel'], g))
        if not self.neg['cos_g_one']:
            assert self.cos_fails(got, CR.head(F['x'], F['w'], F['t'], F['sel'], 1.0)), "negative control: g = 1 passed"
            self.neg['cos_g_one'] += 1
        self.cos['dW'] = dw
        self.cos_dx_readers = {'osb_bn_backward_reduce': dx_a, 'osb_bn_backward_apply': dx_a}
        self.written.add(dx_a)
        return 0

    def cos_gradient_read(self, name, g_a):
        """the first BatchNorm backward reduce / apply after the cosine backward reads its dx as g"""
        want = self.cos_dx_readers.pop(name, None)
        if want is not None:
            assert g_a == want, f"{name}: the first BatchNorm backward does not read the cosine head's dx"


def main():
    kind, arch, scene = cfg.split(':')[:3]
    train = kind in ('train', 'train_all', 'ce', 'cos')
    head = 20 if kind == 'ce' else (int(cfg.split(':')[3]) if kind == 'cos' and cfg.count(':') > 2 else 768)
    model = synth.build_model(arch, head, seed=0).to(dev).train()
    H = Harness(model)
    C.lib = lambda: H
    C.call = H.call
    coords = torch.from_numpy(synth.scene(scene)).to(dev)
    n = coords.shape[0]
    gen = torch.Generator(device=dev).manual_seed(1)
    feats = torch.rand(n, 3, device=dev, generator=gen)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    bns = [nm for nm, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm1d)]
    if kind == 'bs':
        for _ in range(2):
            H.stats.clear()
            with torch.no_grad():
                eng(coords, feats)
            torch.cuda.synchronize()
            assert sorted(s['bn'] for s in H.stats) == sorted(bns), "not exactly one statistics launch per BatchNorm"
    elif kind == 'ce':
        labels = torch.randint(0, 20, (n,), device=dev, generator=gen)
        labels[::9] = 255
        loss, _ = eng.forward_train_ce(coords, feats, labels, 255)
        assert sorted(s['bn'] for s in H.stats) == sorted(bns), "not exactly one statistics launch per BatchNorm"
        loss.backward()
    elif kind == 'cos':
        caller = (torch.arange(n, device=dev) %% 7 == 0).nonzero().squeeze(1)
        feat = torch.randn(caller.numel(), head, device=dev, generator=gen).half()
        H.cos_caller = (caller, feat, 0.75)
        mask = torch.zeros(n, dtype=torch.bool, device=dev)
        mask[caller] = True
        loss = eng.forward_train_cosine(coords, feats, feat, mask)
        assert sorted(s['bn'] for s in H.stats) == sorted(bns), "not exactly one statistics launch per BatchNorm"
        (0.75 * loss).backward()
    else:
        rows_ = None if cfg.endswith(':all') else (torch.arange(n, device=dev) %% 7 == 0)
        out = eng.forward_train(coords, feats, rows=rows_)
        assert sorted(s['bn'] for s in H.stats) == sorted(bns), "not exactly one statistics launch per BatchNorm"
        out.backward(torch.randn(out.shape, device=dev, generator=gen))
    torch.cuda.synchronize()
    if train:
        mods = dict(model.named_modules())
        for nm in bns:
            dw, db = H.reduce_last[nm]
            assert torch.equal(dw, mods[nm].weight.grad) and torch.equal(db, mods[nm].bias.grad), f"{nm}: dweight / dbias not in its gradient slot"
        if kind == 'ce':
            assert torch.equal(H.ce['w_val'], model.final.kernel.detach().view(H.ce['w_val'].shape))
            assert torch.equal(H.ce['dW'], model.final.kernel.grad.view(H.ce['dW'].shape)), "the CE dW is not final.kernel.grad"
        if kind == 'cos':
            assert H.counts['osb_cos_head_fwd'] == H.counts['osb_cos_head_bwd'] == 1, dict(H.counts)
            assert not H.cos_dx_readers, f"no BatchNorm backward read the cosine dx: {sorted(H.cos_dx_readers)}"
            assert torch.equal(H.cos['w'], model.final.kernel.detach().view(H.cos['w'].shape))
            assert torch.equal(H.cos['dW'], model.final.kernel.grad.view(H.cos['dW'].shape)), "the cosine dW is not final.kernel.grad"
        print('SLOTS every BatchNorm\'s dweight / dbias equal its .grad bit for bit', flush=True)
    print('CONFIG', cfg, 'rows', n, 'BatchNorms', len(bns), flush=True)
    print('COUNTS', dict(H.counts), flush=True)
    for op, r in sorted(H.worst.items()):
        print('WORST %%-16s %%.3f of the bound' %% (op, r), flush=True)
    downsample = any(A['res_bn'] for A in H.applies)
    assert H.neg['swapped_form'] == H.neg['own_bn_on_downsample'] == (1 if downsample else 0), dict(H.neg)
    assert H.neg['dropped_mask'] == (1 if train else 0), dict(H.neg)
    cos_neg = [H.neg[k] for k in ('cos_rows_through_perm', 'cos_targets_rolled', 'cos_g_one')]
    assert cos_neg == [1 if kind == 'cos' else 0] * 3, dict(H.neg)
    print('NEGATIVE controls failed as they must:', dict(H.neg), flush=True)
    print('OK')


main()
'''

CONFIGS = [
    'bs:MinkUNet34C:config1_50k',                      # distill's validate(): the batch-statistics forward
    'bs:MinkUNet14A:tiny',                             # coarse levels of a handful of rows
    'train:MinkUNet18A:config1_50k:mask',
    'train:MinkUNet18A:config1_50k:all',
    'ce:MinkUNet18A:config1_50k',
    'cos:MinkUNet34C:config1_50k',                     # the shipped distillation step: 768-wide head on 96 channels
    'cos:MinkUNet14D:config1_50k:512',                 # cin 384: the head's largest shared-memory plan
]
ARCHS = ['MinkUNet14A', 'MinkUNet14B', 'MinkUNet14C', 'MinkUNet14D', 'MinkUNet18A', 'MinkUNet18B', 'MinkUNet18D',
         'MinkUNet34A', 'MinkUNet34B', 'MinkUNet34C']


def _run(cfg, timeout=900):
    r = subprocess.run([sys.executable, '-c', WORKER % {'root': ROOT}, cfg], capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-2500:] + r.stderr[-2500:]


@pytest.mark.parametrize('cfg', CONFIGS)
def test_norm_replay(cfg):
    _run(cfg)


@pytest.mark.parametrize('arch', ARCHS)
def test_norm_replay_every_architecture(arch):
    _run(f'train_all:{arch}:tiny:mask')


@pytest.mark.parametrize('arch', ARCHS)
def test_norm_replay_cosine_every_architecture(arch):
    _run(f'cos:{arch}:tiny')
