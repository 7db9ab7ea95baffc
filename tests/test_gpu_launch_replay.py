"""Every convolution launch of the fused engine replayed in fp64 on the operands it actually read.

The end-to-end tests compare whole networks (1e-3 per point after 60+ layers) and gradients with a yardstick of ~1e-2 of
their largest magnitude (ReLU masks flip under split-row rounding, DESIGN.md section 2): an error below that in one layer --
a missing offset on a tail tile, a wrong transposed pack, a dropped row range -- would pass them.  Here the library seen by
the engine is a wrapper: around every convolution launch it synchronises, snapshots the operands (raw device pointers read
through ``__cuda_array_interface__``), launches the real entry point, snapshots what it wrote and compares that with an fp64
reference of the same operation on the snapshots (tests/replay_ref.py), element by element:

    |y - y^| <= c * 2^-16 * A  (+ 2^-17 |y^| for split outputs),   A = sum |x||W|  (wgrad: sum |x||g|)

with c derived from the kernel's accumulation depth (DESIGN.md section 2).  Packed weights resolve to the fp32 weights they
were packed from through a registry kept by wrapping ``tc.pack_weights`` / ``tc.pack_weight_tiles``.  In training runs each
backward launch is paired with its forward: the weight gradient runs on the forward's map, each input gradient on its exact
transpose with the transposed pack of the same weight slice whose gradient the wgrad produced, and an accumulating input
gradient continues the previous contribution to that source.  Negative controls mutate only the reference side.

Entry points that are neither replayed nor on the pass-through list fail the run, so a launch added to the engine later is
checked or listed on purpose.  Each configuration runs in its own process."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import collections, os, sys, torch
sys.path.insert(0, %(root)r)
cfg = sys.argv[1]
if cfg.endswith('_nochain'):
    os.environ['OSB_CHAIN'] = '0'
from openscene_b200 import engine, synth, tc, _cabi as C
from tests import replay_ref as R

dev = torch.device('cuda:0')

# entry points passed through unreplayed, each owned by another test
PASS = {
    'osb_bn_batch_stats', 'osb_bn_apply_split', 'osb_bn_batch_stats_save', 'osb_bn_apply_split_out',   # test_gpu_norm_replay.py
    'osb_bn_backward_reduce',                                                                           # test_gpu_norm_replay.py
    'osb_bn_stats_workspace_bytes',
    'osb_ce_head_fwd', 'osb_ce_head_bwd', 'osb_ce_head_workspace_bytes',                                # test_gpu_norm_replay.py
    'osb_cos_head_fwd', 'osb_cos_head_bwd', 'osb_cos_head_workspace_bytes',                             # test_gpu_norm_replay.py
    'osb_f32_to_split', 'osb_split_to_f32', 'osb_gather_rows_f32',              # test_gpu_conv_tc.py, test_gpu_engine.py
    'osb_kernel_map_build', 'osb_kernel_map_build_grid', 'osb_kernel_map_transpose', 'osb_hash_build',  # test_gpu_coords.py
    'osb_coordset_build', 'osb_coordset_stride', 'osb_coordset_pyramid', 'osb_coordset_workspace_bytes',
    'osb_occgrid_build', 'osb_occgrid_bytes',
    'osb_folded_head_finish',                                                                           # test_gpu_fast_eval.py
    'osb_conv_pack_weights', 'osb_conv_pack_weight_tiles', 'osb_conv_packed_weight_bytes',   # the packs: registry below,
    'osb_conv_weight_tiles_bytes',                                                           # checked by every replay
    'osb_conv_tc_workspace_bytes', 'osb_conv_chain_workspace_bytes', 'osb_conv_wgrad_tc_workspace_bytes',
    'osb_conv_desc_bytes', 'osb_conv_chain_grid', 'osb_last_error', 'osb_tuning_set',
}
REPLAYED = ('osb_conv_fwd_tc', 'osb_conv_desc_fill', 'osb_conv_chain_launch', 'osb_convtr_fwd_tc', 'osb_conv_stem_fused',
            'osb_conv_stem_fused_grid', 'osb_conv_wgrad_tc', 'osb_conv_fwd_f32', 'osb_bn_backward_apply')


def _i(a):
    return 0 if a is None else (a if isinstance(a, (int, float)) else (a.value or 0))


class _Raw:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (ptr, False), 'version': 3}


def snap(ptr, nbytes):
    return torch.as_tensor(_Raw(ptr, nbytes), device=dev).clone()


def f32(ptr, *shape):
    n = 1
    for s in shape:
        n *= s
    return snap(ptr, 4 * n).view(torch.float32).view(*shape) if ptr else None


def i32(ptr, *shape):
    n = 1
    for s in shape:
        n *= s
    return snap(ptr, 4 * n).view(torch.int32).view(*shape) if ptr else None


class Harness:
    def __init__(self):
        self.real = C.lib()
        self.packs = {}                    # packed address -> (fp32 w3, transpose_w, module ident)
        self.descs = {}                    # host descriptor address -> layer arguments
        self.mods = []                     # (name, kernel3) of every convolution of the model
        self.log = []                      # replayed launches
        self.counts = collections.Counter()
        self.worst = collections.defaultdict(lambda: [0.0, 0.0])     # op -> [worst err / (2^-16 A), c of that launch]
        self.gp = []                       # (gp buffer, accumulate) of osb_bn_backward_apply
        self.neg = collections.Counter()
        self.prev_out = None

    # ---------------------------------------------------------------- weights
    def ident(self, w3, transposed):
        """(module index, lo, form) of the weights a pack was made from, or None (the folded head).  A transposed pack is made
        from the module's own [K, cin, cout] slice, so both forms compare as given."""
        K, c, co = w3.shape
        for mi, (name, k3) in enumerate(self.mods):
            if k3.shape[0] == K and k3.shape[2] == co and k3.shape[1] >= c:
                for lo in range(0, k3.shape[1] - c + 1, 32 if c %% 32 == 0 else 1):
                    if torch.equal(k3[:, lo:lo + c], w3):
                        return (mi, lo, 'plain')
            if K == 1 and k3.shape[0] == 8 and c == k3.shape[1] and co == 8 * k3.shape[2]:
                if torch.equal(k3.permute(1, 0, 2).reshape(1, c, co), w3):
                    return (mi, 0, 'wide')
        return None

    def register(self, fn):
        def wrapped(w3, transpose_w=False):
            out = fn(w3, transpose_w)
            w = w3.detach().contiguous().float().clone()
            self.packs[out.data_ptr()] = (w, bool(transpose_w), self.ident(w, bool(transpose_w)), out)
            return out
        return wrapped

    def weights(self, addr):
        w, t, idt, _ = self.packs[addr]
        return (w.transpose(1, 2) if t else w), t, idt

    # ---------------------------------------------------------------- library wrapper
    def __getattr__(self, name):
        if name in PASS:
            return getattr(self.real, name)
        if name in REPLAYED:
            return getattr(self, '_' + name[4:])
        raise AssertionError(f"entry point {name} is neither replayed nor on the pass-through list")

    def call(self, name, *a):
        C.check(getattr(self, name)(*a), name)

    def check(self, op, y, ref, a, c, split_out=False):
        r = R.worst(y, ref, a, c, split_out)
        w = self.worst[op]
        if r > w[0]:
            w[0], w[1] = r, c
        assert r <= c, f"{op}: error {r:.3g} x 2^-16 A exceeds the bound c = {c:.3g}"
        return r

    # ---------------------------------------------------------------- one convolution layer (osb_conv_fwd_tc or a chain layer)
    def layer(self, L, get, out_get, op):
        """L: argument dict; get(addr, nbytes) reads an input snapshot, out_get(addr, nbytes) an output snapshot"""
        K, cout, n_out = L['K'], L['cout'], L['n_out']
        nbr = i32(L['nbr'], K, n_out) if L['nbr'] else None
        if L.get('cmap'):
            return self.dense_up(L, get, out_get, op)
        n_in = L.get('n_src0') or (int(nbr.max()) + 1 if nbr is not None else n_out)
        xs = [R.split_decode(get(L['src0'], n_in * 4 * L['c0']).view(n_in, -1), L['c0'])]
        if L['src1']:
            n1 = L.get('n_src1') or n_in
            xs.append(R.split_decode(get(L['src1'], n1 * 4 * L['c1']).view(n1, -1), L['c1']))
        x = torch.cat(xs, 1)
        W, T, idt = self.weights(L['wpack'])
        res = R.split_decode(get(L['res'], n_out * 4 * cout).view(n_out, -1), cout) if L['res'] else None
        scale, shift = f32(L['scale'], cout), f32(L['shift'], cout)
        ref, a = R.conv(x, nbr, n_out, W)
        ref, a = R.epilogue(ref, a, scale, shift, res, bool(L['relu']))
        c = R.c_forward(K, x.shape[1])
        tag = op + ('-dgrad' if T else '')
        outs = []
        if L['out_split']:
            y = R.split_decode(out_get(L['out_split'], n_out * 4 * cout).view(n_out, -1), cout)
            self.check(tag, y, ref, a, c, split_out=True)
            outs.append(y)
        if L['out_f32']:
            rm = i32(L['row_map'], n_out) if L['row_map'] else None
            rows = int(rm.max()) + 1 if rm is not None else n_out
            y = out_get(L['out_f32'], rows * 4 * cout).view(torch.float32).view(rows, cout)
            y = y[rm.long()] if rm is not None else y
            if rm is not None:
                assert torch.unique(rm).numel() == n_out
            self.check(tag, y, ref, a, c)
            outs.append(y.double())
        self.negatives(L, x, nbr, n_out, W, T, scale, shift, res, outs[0], ref, a, c)
        self.log.append(dict(op='fwd', T=T, idt=idt, nbr=nbr, n_out=n_out, n_in=n_in, src=[L['src0'], L['src1']], widths=[L['c0'], L['c1']],
                             res=L['res'], out=L['out_split'] or L['out_f32'], cmap=None))

    def dense_up(self, L, get, out_get, op):
        cmap = i32(L['cmap'], 8, L['n_out'])
        n_c, cout = L['n_out'], L['cmap_cout']
        n_f = int((cmap >= 0).sum())
        x = R.split_decode(get(L['src0'], n_c * 4 * L['c0']).view(n_c, -1), L['c0'])
        wide, T, idt = self.weights(L['wpack'])
        w = wide[0].view(L['c0'], 8, cout).permute(1, 0, 2)
        ref, a = R.convtr(x, cmap, w, n_f)
        ref, a = R.epilogue(ref, a, f32(L['scale'], cout), f32(L['shift'], cout), None, bool(L['relu']))
        c = R.c_forward(1, L['c0'])
        if L['out_split']:
            self.check(op + '-up', R.split_decode(out_get(L['out_split'], n_f * 4 * cout).view(n_f, -1), cout), ref, a, c, True)
        if L['out_f32']:
            self.check(op + '-up', out_get(L['out_f32'], n_f * 4 * cout).view(torch.float32).view(n_f, cout), ref, a, c)
        self.log.append(dict(op='fwd', T=False, idt=idt, nbr=R.transpose_map(cmap, n_f), n_out=n_f, n_in=n_c, src=[L['src0'], 0],
                             widths=[L['c0'], 0], res=0, out=L['out_split'] or L['out_f32'], cmap=cmap))

    def negatives(self, L, x, nbr, n_out, W, T, scale, shift, res, y, ref, a, c):
        """mutations of the reference side only: each must fail the bound"""
        def fails(y_, ref_, a_):
            return R.worst(y_, ref_, a_, c) > c
        if not self.neg['tile'] and nbr is not None and W.shape[0] == 27 and n_out > 256 and not T:
            m = nbr.clone()
            m[13, 128:256] = -1                       # the centre offset (always present) dropped for one 128-row tile
            r2, a2 = R.epilogue(*R.conv(x, m, n_out, W), scale, shift, res, bool(L['relu']))
            assert fails(y, r2, a2), "negative control: a dropped offset tile was not detected"
            self.neg['tile'] += 1
        if not self.neg['transpose'] and T and W.shape[1] == W.shape[2]:
            r2, a2 = R.epilogue(*R.conv(x, nbr, n_out, W.transpose(1, 2)), scale, shift, res, bool(L['relu']))
            assert fails(y, r2, a2), "negative control: a flipped transpose_w was not detected"
            self.neg['transpose'] += 1
        if not self.neg['stale'] and self.prev_out is not None and self.prev_out.shape == y.shape:
            assert fails(self.prev_out, ref, a), "negative control: the previous launch's output passed as this one's"
            self.neg['stale'] += 1
        self.prev_out = y

    # ---------------------------------------------------------------- entry points
    def _conv_fwd_tc(self, *args):
        a = [_i(v) for v in args]
        L = dict(src0=a[0], c0=a[1], n_src0=a[2], src1=a[3], c1=a[4], n_src1=a[5], nbr=a[6], n_out=a[7], K=a[8], wpack=a[9], cout=a[10],
                 scale=a[11], shift=a[12], res=a[13], relu=a[14], out_split=a[15], out_f32=a[16], row_map=a[17], cmap=0, cmap_cout=0)
        return self._group('osb_conv_fwd_tc', [L], lambda: self.real.osb_conv_fwd_tc(*args), 'conv_fwd_tc')

    def _conv_desc_fill(self, *args):
        a = [_i(v) for v in args]
        self.descs[a[0]] = dict(src0=a[1], c0=a[2], src1=a[3], c1=a[4], nbr=a[5], n_out=a[6], K=a[7], wpack=a[8], cout=a[9],
                                scale=a[10], shift=a[11], res=a[12], relu=a[13], out_split=a[14], out_f32=a[15], row_map=a[16],
                                cmap=a[17], cmap_cout=a[18])
        return self.real.osb_conv_desc_fill(*args)

    def _conv_chain_launch(self, *args):
        a = [_i(v) for v in args]
        db = self.real.osb_conv_desc_bytes()
        layers = [dict(self.descs[a[0] + i * db]) for i in range(a[1])]
        self.counts['chain layer'] += len(layers)
        return self._group('osb_conv_chain_launch', layers, lambda: self.real.osb_conv_chain_launch(*args), 'chain')

    def _convtr_fwd_tc(self, *args):
        a = [_i(v) for v in args]
        assert a[4] == 8
        L = dict(src0=a[0], c0=a[1], n_out=a[2], cmap=a[3], K=1, wpack=a[5], cmap_cout=a[6], cout=8 * a[6], scale=a[7],
                 shift=a[8], relu=a[9], out_split=a[10], out_f32=a[11], nbr=0, src1=0, c1=0, res=0, row_map=0)
        return self._group('osb_convtr_fwd_tc', [L], lambda: self.real.osb_convtr_fwd_tc(*args), 'convtr_fwd_tc')

    def _group(self, name, layers, launch, op):
        """snapshot every input of a launch, launch, snapshot every output, replay each layer in order"""
        torch.cuda.synchronize()
        written, size = set(), {}
        for L in layers:
            for k in ('out_split', 'out_f32'):
                if L[k]:
                    assert L[k] not in written, "a buffer written twice within one launch: the replay could not be faithful"
                    written.add(L[k])
            K, n_out = L['K'], L['n_out']
            if 'n_src0' not in L:                        # chain layers: input rows from the map
                if L['cmap']:
                    n_in = n_out
                else:
                    nbr = i32(L['nbr'], K, n_out) if L['nbr'] else None
                    n_in = int(nbr.max()) + 1 if nbr is not None else n_out
                L['n_src0'] = L['n_src1'] = n_in
            for k, c, rows in (('src0', L['c0'], L['n_src0']), ('src1', L['c1'], L.get('n_src1')), ('res', L['cout'], n_out)):
                if L[k]:
                    size[L[k]] = max(size.get(L[k], 0), rows * 4 * c)
        pre = {p: snap(p, nb) for p, nb in size.items()}
        rc = launch()
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts[name] += 1
        post, done = {}, set()
        for L in layers:
            rows = int((i32(L['cmap'], 8, L['n_out']) >= 0).sum()) if L['cmap'] else L['n_out']
            oc = L['cmap_cout'] if L['cmap'] else L['cout']
            if L['out_split']:
                post[L['out_split']] = snap(L['out_split'], rows * 4 * oc)
            if L['out_f32']:
                rm = i32(L['row_map'], L['n_out']) if L['row_map'] else None
                post[L['out_f32']] = snap(L['out_f32'], (int(rm.max()) + 1 if rm is not None else rows) * 4 * oc)
        for L in layers:
            # an input an earlier layer of this launch wrote is read after that layer: its post-launch snapshot
            get = lambda p, nb: (post[p] if p in done else pre[p])[:nb]
            self.layer(L, get, lambda p, nb: post[p][:nb], op)
            done.update(x for x in (L['out_split'], L['out_f32']) if x)
        return 0

    def _stem(self, name, args, grid):
        a = [_i(v) for v in args]
        cin, n = a[1], a[3]
        ks, step, w_a, cout = (a[8], a[9], a[10], a[11]) if grid else (a[6], a[7], a[8], a[9])
        scale_a, shift_a, relu, os_, of_ = a[-6:-1]
        torch.cuda.synchronize()
        x = f32(a[0], n, cin).double()
        coords = i32(a[2], n, 4)
        w = f32(w_a, ks ** 3, cin, cout)
        rc = getattr(self.real, name)(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts[name] += 1
        nbr = R.neighbour_map(coords, ks, step)                # independent of the library's hash / grid
        ref, A = R.conv(x, nbr, n, w)
        ref, A = R.epilogue(ref, A, f32(scale_a, cout), f32(shift_a, cout), None, bool(relu))
        c = R.c_fma(ks ** 3 * cin)
        if os_:
            self.check('stem', R.split_decode(snap(os_, n * 4 * cout).view(n, -1), cout), ref, A, c, True)
        if of_:
            self.check('stem', f32(of_, n, cout), ref, A, c)
        self.log.append(dict(op='fwd', T=False, idt=self.ident(w, False), nbr=nbr, n_out=n, n_in=n, src=[a[0], 0], widths=[cin, 0],
                             res=0, out=os_ or of_, cmap=None, stem=True))
        return 0

    def _conv_stem_fused(self, *args):
        return self._stem('osb_conv_stem_fused', args, False)

    def _conv_stem_fused_grid(self, *args):
        return self._stem('osb_conv_stem_fused_grid', args, True)

    def _conv_wgrad_tc(self, *args):
        a = [_i(v) for v in args]
        x_a, cin, n_in, nbr_a, n_out, K, g_a, cout, gw_a = a[:9]
        torch.cuda.synchronize()
        x = R.split_decode(snap(x_a, n_in * 4 * cin).view(n_in, -1), cin)
        nbr = i32(nbr_a, K, n_out) if nbr_a else None
        g = R.split_decode(snap(g_a, n_out * 4 * cout).view(n_out, -1), cout)
        rc = self.real.osb_conv_wgrad_tc(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_conv_wgrad_tc'] += 1
        gw = f32(gw_a, K, cin, cout)
        ref, A = R.wgrad(x, nbr, g, K)
        c = R.c_wgrad(n_out, K, cin, cout)
        self.check('wgrad', gw, ref, A, c)
        self.log.append(dict(op='wgrad', x=x_a, gout=g_a, nbr=nbr, n_rs=R.wgrad_plan(n_out, K, cin, cout)[0], gw=gw, K=K))
        return 0

    def _conv_fwd_f32(self, *args):
        a = [_i(v) for v in args]
        in_a, ld, nbr_a, n_out, K, w_a, cin, cout, tw, out_a = a[:10]
        assert not nbr_a and K == 1 and ld == cin and not tw
        torch.cuda.synchronize()
        x = f32(in_a, n_out, cin).double()
        w = f32(w_a, 1, cin, cout)
        rc = self.real.osb_conv_fwd_f32(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_conv_fwd_f32'] += 1
        ref, A = R.conv(x, None, n_out, w)
        self.check('conv_fwd_f32', f32(out_a, n_out, cout), ref, A, R.c_fma(cin))
        self.log.append(dict(op='fwd', T=False, idt=self.ident(w, False), nbr=None, n_out=n_out, n_in=n_out, src=[in_a, 0],
                             widths=[cin, 0], res=0, out=out_a, cmap=None))
        return 0

    def _bn_backward_apply(self, *args):
        a = [_i(v) for v in args]
        if a[10]:
            self.gp.append((a[10], a[11]))
        return self.real.osb_bn_backward_apply(*args)


def pairing(H, model, head_launch):
    """each backward launch against the forward it differentiates"""
    fwd = [r for r in H.log if r['op'] == 'fwd' and not r['T']]
    dgr = [(i, r) for i, r in enumerate(H.log) if r['op'] == 'fwd' and r['T']]
    wgr = [(i, r) for i, r in enumerate(H.log) if r['op'] == 'wgrad']
    by_mod = collections.defaultdict(list)
    for r in fwd:
        if r['idt'] is not None:
            by_mod[r['idt'][0]].append(r)
    names = [n for n, _ in H.mods]
    for mi, name in enumerate(names):
        if head_launch and name == 'final':
            continue                                   # the head's forward is osb_ce_head_fwd / osb_cos_head_fwd
        assert len(by_mod[mi]) == 1, f"{name}: {len(by_mod[mi])} forward launches"
    latest, gp_bufs, n_pairs = {}, {b for b, acc in H.gp if not acc}, 0
    used = set()
    for i, D in dgr:
        mi, lo, form = D['idt']
        assert form == 'plain', "a dgrad pack that is not W^T of a module slice"
        F = by_mod[mi][0]
        s = 0 if lo == 0 else 1
        assert lo == (0 if s == 0 else F['widths'][0]) and D['widths'][0] == H.mods[mi][1].shape[2]
        assert D['n_out'] == F['n_in']
        x_src = F['src'][s]
        W = [r for j, r in wgr if j < i and r['gout'] == D['src'][0] and r['x'] == x_src]
        assert W, f"{names[mi]}: no weight gradient over the dgrad's output gradient and the forward's source {s}"
        W = W[-1]
        fmap = F['nbr']
        assert (W['nbr'] is None) == (fmap is None) and (fmap is None or torch.equal(W['nbr'].long(), fmap.long())), \
            f"{names[mi]}: the weight gradient does not run on the forward's map"
        if fmap is None:
            assert D['nbr'] is None, f"{names[mi]}: identity forward, mapped dgrad"
        else:
            assert torch.equal(D['nbr'].long(), R.transpose_map(fmap.long(), D['n_out'])), \
                f"{names[mi]}: the dgrad map is not the exact transpose of the forward map"
            if F['cmap'] is not None:
                assert torch.equal(D['nbr'], F['cmap'])
        k3 = H.mods[mi][1]
        grad = dict(model.named_modules())[names[mi]].kernel.grad
        grad = grad.view(k3.shape)
        assert torch.equal(W['gw'], grad[:, lo:lo + W['gw'].shape[1]]), f"{names[mi]}: the wgrad result is not the slot of slice {lo}"
        # accumulation: a dgrad with a residual continues the previous contribution to the same source
        if D['res']:
            assert D['res'] == latest.get(x_src, D['res'] if D['res'] in gp_bufs else -1), \
                f"{names[mi]}: the accumulating dgrad does not read the previous contribution to its source"
        else:
            assert x_src not in latest, f"{names[mi]}: a second contribution to a source overwrites the first"
        latest[x_src] = D['out']
        used.add(id(W))
        n_pairs += 1
    # every kernel received a weight gradient: the stem's padded one, and one per source of [up | skip] inputs
    for mi, (name, k3) in enumerate(H.mods):
        if head_launch and name == 'final':
            continue
        grad = dict(model.named_modules())[name].kernel.grad.view(k3.shape)
        F = by_mod[mi][0]
        widths = [w for w in F['widths'] if w]
        lo = 0
        for w in widths:
            hit = [r for _, r in wgr if r['gw'].shape[0] == k3.shape[0] and r['gw'].shape[2] == k3.shape[2]
                   and r['gw'].shape[1] >= w and torch.equal(r['gw'][:, :w], grad[:, lo:lo + w])]
            assert hit, f"{name}: no weight gradient for input channels {lo}:{lo + w}"
            lo += w
    return n_pairs


def main():
    parts = cfg.split(':')
    kind, arch, scene = parts[0], parts[1], parts[2]
    H = Harness()
    C.lib = lambda: H
    C.call = H.call
    tc._CHAINS.clear()
    tc._PACK_CACHE.clear()
    tc.pack_weights = H.register(tc.pack_weights)
    tc.pack_weight_tiles = H.register(tc.pack_weight_tiles)
    train = kind in ('train', 'train_all', 'ce', 'cos')
    head = 20 if kind in ('ce', 'eval20') else 768
    model = synth.build_model(arch, head, seed=0).to(dev)
    model.train() if train else model.eval()
    H.mods = [(n, (m.kernel.detach().unsqueeze(0) if m.kernel.dim() == 2 else m.kernel.detach()).float().clone())
              for n, m in model.named_modules() if hasattr(m, 'kernel') and isinstance(m.kernel, torch.nn.Parameter)]
    coords = torch.from_numpy(synth.scene(scene)).to(dev)
    n = coords.shape[0]
    gen = torch.Generator(device=dev).manual_seed(1)
    feats = torch.rand(n, 3, device=dev, generator=gen)
    eng = engine.FusedMinkUNet(model, batch_stats=train)
    names = [nm for nm, _ in H.mods]

    def coverage(skip_final):
        """every convolution kernel in exactly one forward replay of this run"""
        seen = collections.Counter(r['idt'][0] for r in H.log if r['op'] == 'fwd' and not r['T'] and r['idt'] is not None)
        for mi, nm in enumerate(names):
            assert seen[mi] == (0 if (skip_final and nm == 'final') else 1), (nm, seen[mi])
        print('COVERAGE forward: every one of', len(names) - skip_final, 'kernels in exactly one forward replay', flush=True)

    if kind.startswith('eval'):
        eng(coords, feats)
        coverage(False)
        if cfg.endswith('_nochain'):
            H.log.clear()
            folded = eng.fold_head(torch.from_numpy(synth.text_embeddings(20)).float().to(dev))
            eng.forward_scores(coords, feats, folded)
            coverage(True)
    elif kind == 'ce':
        labels = torch.randint(0, 20, (n,), device=dev, generator=gen)
        labels[::9] = 255
        loss, _ = eng.forward_train_ce(coords, feats, labels, 255)
        loss.backward()
        coverage(True)
    elif kind == 'cos':
        mask = torch.arange(n, device=dev) %% 7 == 0
        feat = torch.randn(int(mask.sum()), 768, device=dev, generator=gen).half()
        loss = eng.forward_train_cosine(coords, feats, feat, mask)
        (0.75 * loss).backward()
        coverage(True)
    else:
        rows = None if parts[3] == 'all' else (torch.arange(n, device=dev) %% 7 == 0)
        out = eng.forward_train(coords, feats, rows=rows)
        out.backward(torch.randn(out.shape, device=dev, generator=gen))
        coverage(False)
    torch.cuda.synchronize()
    print('CONFIG', cfg, 'rows', n, flush=True)
    print('COUNTS', dict(H.counts), flush=True)
    for op, (r, c) in sorted(H.worst.items()):
        print('WORST %%-22s err/A = %%.3f x 2^-16   (bound c = %%.1f)' %% (op, r, c), flush=True)
    if train:
        pairs = pairing(H, model, kind in ('ce', 'cos'))
        print('PAIRING', pairs, 'dgrad launches paired with their forward and weight gradient; every kernel has its wgrads;',
              'n_rs > 1 in', sum(1 for r in H.log if r['op'] == 'wgrad' and r['n_rs'] > 1), 'wgrads', flush=True)
    assert H.neg['tile'] == 1 and H.neg['stale'] == 1 and (H.neg['transpose'] == 1 or not train), dict(H.neg)
    print('NEGATIVE controls failed the bound as they must:', dict(H.neg), flush=True)
    print('OK')


main()
'''

CONFIGS = [
    'eval:MinkUNet34C:config2_200k',                   # bench.py's workload: the persistent chain
    'eval:MinkUNet34C:config2_200k:_nochain',          # osb_conv_fwd_tc + osb_convtr_fwd_tc, and forward_scores' folded head
    'eval20:MinkUNet18A:tiny',                         # a 20-class head: osb_conv_fwd_f32
    'train:MinkUNet18A:config1_50k:mask',
    'train:MinkUNet34C:config1_50k:mask',
    'train:MinkUNet18A:tiny:all',
    'ce:MinkUNet18A:config1_50k',
    'cos:MinkUNet34C:config1_50k:mask',                # the cosine distillation step: the trunk under osb_cos_head_*
    'cos:MinkUNet18A:tiny:mask',
]
ARCHS = ['MinkUNet14A', 'MinkUNet14B', 'MinkUNet14C', 'MinkUNet14D', 'MinkUNet18A', 'MinkUNet18B', 'MinkUNet18D',
         'MinkUNet34A', 'MinkUNet34B', 'MinkUNet34C']


def _run(cfg, timeout=1200):
    r = subprocess.run([sys.executable, '-c', WORKER % {'root': ROOT}, cfg], capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-5000:], r.stderr[-3000:])
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout[-2500:] + r.stderr[-2500:]


@pytest.mark.parametrize('cfg', CONFIGS)
def test_launch_replay(cfg):
    _run(cfg)


@pytest.mark.parametrize('arch', ARCHS)
def test_launch_replay_every_architecture(arch):
    _run(f'train_all:{arch}:tiny:mask')
