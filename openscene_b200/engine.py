"""Fused inference engine for the MinkUNet family (eval mode) on libosb200.

Takes a network built from the MinkowskiEngine surface (``openscene_b200.minkunet.MinkUNet`` or the
reference's own ``models/mink_unet.py`` classes running on this repository's ``MinkowskiEngine``
package) and executes ``MinkUNetBase.forward`` (models/mink_unet.py:116-174) as one C-ABI call per
convolution:

* BatchNorm (eval) is folded into the producing convolution's epilogue (scale/shift), ReLU and the
  BasicBlock residual add likewise; ``ME.cat`` is never materialised (the next convolution reads two
  sources); activations stay in the split-bf16 layout between layers;
* the 5x5x5 stem fuses its 125 neighbour lookups (occupancy grid, or the hash where that does not fit) with the 3->32 FMA
  (no 5^3 kernel map in HBM);
* the final 1x1x1 convolution writes fp32 rows straight into the caller's row order.

Results equal the module-by-module path within the bf16x3 tolerance (tests/test_gpu_engine.py).

``FusedMinkUNet(model, batch_stats=True)`` runs a TRAIN-mode network instead (the forward run/distill.py's validate() makes
under no_grad): every BatchNorm normalises with the statistics of the current batch and moves its running buffers as
``nn.BatchNorm1d`` does.  Each convolution then writes raw rows, ``osb_bn_batch_stats`` reduces them and
``osb_bn_apply_split`` normalises them in place, with the ReLU and the BasicBlock residual (the downsample branch's raw output
is normalised inside that same pass).  Layers run one launch each (a full reduction separates a layer from its consumer, so
the persistent chain has nothing to fuse) (tests/test_gpu_bn_batch_stats.py).

``FusedMinkUNet(model, batch_stats=True, process_group=pg)`` trains data-parallel over ``pg`` as DistributedDataParallel does
with its defaults: rank 0's parameters and buffers are broadcast at construction, its BatchNorm running buffers before a
forward that follows a grad-enabled one, and the backward all-reduces the averaged gradients in buckets while it runs
(engine_train.py).
"""
import os
import zlib

import torch
import torch.distributed as dist

from . import _cabi as C
from . import tc
from .coords import CoordinateManager


def _al(x):
    return (x + 255) & ~255


def _fold_bn(bn_module):
    bn = bn_module.bn
    scale = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).float().contiguous()
    shift = (bn.bias - bn.running_mean * scale).float().contiguous()
    return scale, shift


class _Conv:
    """Packed weights + folded BN of one convolution (batch-statistics mode: the BatchNorm module instead, ``bn``)."""
    __slots__ = ('K', 'cin', 'cout', 'wpack', 'w3', 'scale', 'shift', 'ks', 'stride', 'transpose', 'wpack_a', 'scale_a', 'shift_a',
                 'wtiles', 'wtiles_a', 'n_ntiles', 'bn', 'bs_args', 'bs_scale_a', 'bs_shift_a', 'mod', 'bs_mean_a', 'bs_invstd_a',
                 'bwd')

    def __init__(self, conv, bn=None, keep_f32=False, fold=True):
        if getattr(conv, 'bias', None) is not None:
            raise NotImplementedError("FusedMinkUNet: convolutions with bias are not folded (no MinkUNet layer has one: "
                                      "models/mink_unet.py builds every convolution with bias=False)")
        w3 = conv.kernel.detach()
        w3 = w3.unsqueeze(0) if w3.dim() == 2 else w3
        self.K, self.cin, self.cout = w3.shape
        self.ks, self.stride = conv.kernel_size, conv.stride
        self.transpose = conv.TRANSPOSE
        self.mod, self.bwd = conv, None          # training: the module (parameter -> gradient slot), W^T packs for dgrad
        self.w3 = w3.float().contiguous() if keep_f32 else None
        self.wpack = tc.pack_weights(w3) if (self.cin % 32 == 0 and self.cout % 32 == 0) else None
        self.scale, self.shift = _fold_bn(bn) if (bn is not None and fold) else (None, None)
        self.bn = bn.bn if (bn is not None and not fold) else None
        # raw device addresses for the low-overhead launch path (tensors above keep the memory alive)
        self.wpack_a = self.wpack.data_ptr() if self.wpack is not None else 0
        self.wtiles = tc.pack_weight_tiles(w3) if self.wpack is not None else None        # persistent-kernel packing
        self.wtiles_a = self.wtiles.data_ptr() if self.wtiles is not None else 0
        self.n_ntiles = max(1, -(-self.cout // 128))
        self.scale_a = self.scale.data_ptr() if self.scale is not None else 0
        self.shift_a = self.shift.data_ptr() if self.shift is not None else 0


_BROADCAST_BUCKET_BYTES = 250 << 20               # DistributedDataParallel's broadcast_bucket_size


class FusedMinkUNet:
    def __init__(self, model, batch_stats=False, process_group=None):
        """model: eval-mode MinkUNet (BasicBlock variants) whose parameters live on a CUDA device.
        batch_stats=True: a train-mode model instead; every forward normalises with batch statistics and updates the BatchNorm
        running buffers in place, as ``model(sinput)`` in train mode under no_grad does.
        process_group (batch_stats only): train data-parallel over this group as ``DistributedDataParallel(model)`` does;
        every rank must build its engine, run the same number of forwards and backwards, and pass the same group."""
        net = model.net3d if hasattr(model, 'net3d') else model
        p = next(net.parameters())
        C.require_cuda(p, 'model parameters')
        self.batch_stats = bool(batch_stats)
        if process_group is not None and not self.batch_stats:
            raise ValueError("FusedMinkUNet: process_group needs batch_stats=True (the eval engine computes no gradients to "
                             "all-reduce)")
        self._net = net
        self._check_mode()
        self.device = p.device
        self.process_group = process_group
        self._sync_buffers = True                 # DDP's require_forward_param_sync: broadcast buffers before the next forward
        if process_group is not None:
            self._dp_sync_module_states()         # before anything is packed from the parameters
        self.dense_up = os.environ.get('OSB_DENSE_UP', '1') != '0'
        # The packed weights and folded BatchNorm constants are COPIES: every tensor they were made from is tracked, and a
        # forward that finds one changed (load_state_dict, an optimiser step, .to()) re-packs before it runs.  With batch
        # statistics the running buffers are not copied (the kernels read and update the module's own), see _signature.
        self._tracked = list(net.parameters()) + ([] if self.batch_stats else list(net.buffers()))
        self._bs_ws = None
        self._gen = 0                             # bumped by every forward: a training graph whose activations were overwritten
        self._garena = []                         # training: grow-only chunks of gradient rows (engine_train.py)
        self._ce_ws = None                        # workspace of the CE, cosine and L1 heads (engine_train.py, forward_eval_ce)
        self._build()
        self.out_channels = self.final.cout
        self.last_cm = None
        self._ws = None
        self._arena = None
        self.use_pdl = os.environ.get('OSB_PDL', '1') != '0'
        # persistent chain kernel (csrc/conv_chain.cu); OSB_CHAIN=0 restores one launch of the first-generation kernel per layer
        self.use_chain = os.environ.get('OSB_CHAIN', '1') != '0'
        self.chain_max_tiles = int(os.environ.get('OSB_CHAIN_MAX_TILES', '-1'))   # layers up to this many (row x N) tiles share a launch
        self._chain = None
        self.layer_log = None                     # profiling: set to [] to record (rows, K, cin, cout, tag) per convolution
        self.use_pyramid = os.environ.get('OSB_PYRAMID', '1') != '0'
        if 'OSB_TC_LAZY' in os.environ:                      # tuning: 0 = smem index prologue, 1 = lazy on >= 2-wave launches, 2 = always
            tc.debug_set_tc(lazy=int(os.environ['OSB_TC_LAZY']))

    def _dp_sync_module_states(self):
        """DistributedDataParallel's construction: refuse a model whose parameters differ in count or shape on any rank (on
        every rank, instead of a later collective hanging), then broadcast rank 0's parameters and buffers in place."""
        pg, net = self.process_group, self._net
        params = list(net.parameters())
        shapes = repr([(tuple(p.shape), str(p.dtype)) for p in params]).encode()
        sig = torch.tensor([len(params), sum(p.numel() for p in params), zlib.crc32(shapes)], dtype=torch.int64,
                           device=self.device)
        got = [torch.empty_like(sig) for _ in range(dist.get_world_size(group=pg))]
        dist.all_gather(got, sig, group=pg)
        bad = [r for r, g in enumerate(got) if not torch.equal(g, got[0])]
        if bad:
            raise RuntimeError(f"FusedMinkUNet: the models of process_group ranks {bad} differ from rank 0's in parameter count "
                               f"or shapes ({int(sig[0])} parameters on this rank, rank {dist.get_rank(group=pg)})")
        with torch.no_grad():
            dist._broadcast_coalesced(pg, params + list(net.buffers()), _BROADCAST_BUCKET_BYTES, 0)

    def _dp_forward(self, fn, *args):
        """fn(*args) under DistributedDataParallel's buffer rule (broadcast_buffers=True): rank 0's running buffers are
        broadcast into every rank's storage before the first forward and before any forward that follows a grad-enabled one."""
        if self.process_group is None:
            return fn(*args)
        sync_next = torch.is_grad_enabled()
        if self._sync_buffers:
            with torch.no_grad():
                dist._broadcast_coalesced(self.process_group, [b for m in self._bns for b in
                                                               (m.running_mean, m.running_var, m.num_batches_tracked)],
                                          _BROADCAST_BUCKET_BYTES, 0)
        out = fn(*args)
        self._sync_buffers = sync_next
        return out

    def _check_mode(self):
        if self.batch_stats:
            if not self._net.training or not all(m.training for m in self._net.modules()
                                                 if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)):
                raise RuntimeError("FusedMinkUNet(batch_stats=True) normalises with batch statistics (train-mode BatchNorm): "
                                   "call model.train() first")
        elif self._net.training:
            raise RuntimeError("FusedMinkUNet folds BatchNorm running statistics: call model.eval() first")

    def _signature(self):
        # ~20 us for the 373 tensors of MinkUNet34C: in-place updates (optimiser steps, load_state_dict) bump `_version`; a
        # re-allocation (.to(), assign=True) moves the first / last tensor along with all others
        t = self._tracked
        if self.batch_stats:
            # weights and BatchNorm affine parameters by version; the running buffers only by address: the engine moves them
            # itself every forward, which must not cost a re-pack, but a re-assigned buffer must be picked up
            return (sum(x._version for x in t), tuple(x.data_ptr() for x in t),
                    tuple(b.data_ptr() for m in self._bns for b in (m.running_mean, m.running_var, m.num_batches_tracked)))
        return (sum(x._version for x in t), t[0].data_ptr(), t[-1].data_ptr(), len(t))

    def refresh(self):
        """Re-pack the weights and re-fold BatchNorm from the source module (called automatically when a tracked tensor changed)."""
        self._check_mode()
        self._tracked = list(self._net.parameters()) + ([] if self.batch_stats else list(self._net.buffers()))
        self._build()

    def repack_jobs(self):
        """Batch-statistics engine: [(weight, pack, (sk, sn, sc), K, cin, cout, cout_pad)], one ``osb_conv_repack`` job per
        split-bf16 operand its forwards and backward read, made from the module's current weights (openscene_b200/optim.py
        re-packs them in place after an optimiser step): the forward pack of every convolution, read as the dense-up
        ``[1, cin, K * cout]`` matrix for the transposed ones; the final layer's pack; every per-source ``W^T`` pack the
        backward has built so far.  The stem and the cross-entropy head multiply the parameter itself (``w3`` is the
        parameter's storage) and the persistent-chain tiles are never read with batch statistics."""
        if not self.batch_stats:
            raise RuntimeError("repack_jobs: an eval-mode engine folds BatchNorm into its packs; it re-packs through refresh()")
        jobs = []
        for cv in (self.stem, self.final):
            if cv.w3.data_ptr() != cv.mod.kernel.data_ptr():
                raise RuntimeError("repack_jobs: the engine's fp32 weight copy is not the parameter's storage (refresh first)")
        convs = [(c0, False) for (c0, _) in self.enc] + [(c0, self.dense_up) for (c0, _) in self.dec]
        convs += [(cv, False) for (_, blocks) in self.enc + self.dec for blk in blocks for cv in blk if cv is not None]
        convs.append((self.final, False))
        for cv, wide in convs:
            w = cv.mod.kernel.detach()
            K, cin, cout = cv.K, cv.cin, cv.cout
            if cv.wpack is not None:
                # [K, cin, cout]: element (k, n, c) = W[k, c, n]; the dense-up pack's row k * cout + n is that same element
                pad = cout if wide else cv.wpack.numel() // (4 * K * cin)
                jobs.append((w, cv.wpack, (cin * cout, 1, cout), K, cin, cout, pad))
            if isinstance(cv.bwd, list):
                for (lo, hi, pk) in cv.bwd:                  # W[:, lo:hi, :]^T: element (k, n, c) = W[k, lo + n, c]
                    jobs.append((w[:, lo:hi] if w.dim() == 3 else w[lo:hi], pk, (cin * cout, cout, 1), K, cout, hi - lo,
                                 pk.numel() // (4 * K * cout)))
        return jobs

    def _build(self):
        net = self._net
        fold = not self.batch_stats
        with torch.cuda.device(self.device), torch.no_grad():
            self.stem = _Conv(net.conv0p1s1, net.bn0, keep_f32=True, fold=fold)
            if self.stem.cin > 3 or self.stem.cout != 32:
                raise NotImplementedError("fused stem supports cin <= 3, cout == 32 (every MinkUNet: INIT_DIM = 32, 3 input features)")
            self.enc, self.dec = [], []
            for i in range(1, 5):
                down = _Conv(getattr(net, f'conv{i}p{2 ** (i - 1)}s2'), getattr(net, f'bn{i}'), fold=fold)
                self.enc.append((down, self._blocks(getattr(net, f'block{i}'), fold)))
            for j in range(4, 8):
                m = getattr(net, f'convtr{j}p{2 ** (8 - j)}s2')
                up = _Conv(m, getattr(net, f'bntr{j}'), fold=fold)
                if self.dense_up and up.wpack is not None:
                    # dense transposed conv: one [cin, 8*cout] matrix, column block k = W[k]
                    wide = m.kernel.detach().permute(1, 0, 2).reshape(1, up.cin, up.K * up.cout).contiguous()
                    up.wpack = tc.pack_weights(wide)
                    up.wpack_a = up.wpack.data_ptr()
                    up.wtiles = tc.pack_weight_tiles(wide)
                    up.wtiles_a = up.wtiles.data_ptr()
                    up.n_ntiles = max(1, -(-(up.K * up.cout) // 128))
                self.dec.append((up, self._blocks(getattr(net, f'block{j + 1}'), fold)))
            self.final = _Conv(net.final, None, keep_f32=True)
            if self.batch_stats:
                self._bs_setup()
        self._sig = self._signature()

    @staticmethod
    def _blocks(seq, fold=True):
        out = []
        for b in seq:
            if not hasattr(b, 'conv2') or hasattr(b, 'conv3'):
                raise NotImplementedError("FusedMinkUNet supports BasicBlock networks (all MinkUNet14/18/34 variants)")
            ds = _Conv(b.downsample[0], b.downsample[1], fold=fold) if b.downsample is not None else None
            out.append((_Conv(b.conv1, b.norm1, fold=fold), _Conv(b.conv2, b.norm2, fold=fold), ds))
        return out

    def _bs_setup(self):
        """Batch-statistics mode: one engine-owned fp32 buffer holds the scale / shift of every BatchNorm (written by
        osb_bn_batch_stats, read by osb_bn_apply_split); the kernels update the module's running buffers in place."""
        convs = [self.stem]
        for (c0, blocks) in self.enc + self.dec:
            convs.append(c0)
            convs += [cv for blk in blocks for cv in blk if cv is not None]
        for cv in convs:
            bn = cv.bn
            if not (bn.affine and bn.track_running_stats):
                raise NotImplementedError("FusedMinkUNet(batch_stats=True): BatchNorm without affine parameters or running "
                                          "statistics is not supported (every MinkUNet BatchNorm has both)")
            if (any(t.dtype != torch.float32 for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
                    or bn.num_batches_tracked.dtype != torch.int64):
                raise NotImplementedError("FusedMinkUNet(batch_stats=True): BatchNorm parameters and running statistics must be "
                                          "fp32 (num_batches_tracked int64)")
        # per BatchNorm: scale, shift and (forward_train) the batch mean / invstd the backward reads
        self._bs_buf = torch.empty(sum(4 * cv.cout for cv in convs), dtype=torch.float32, device=self.device)
        a = self._bs_buf.data_ptr()
        for cv in convs:
            bn = cv.bn
            cv.bs_scale_a, cv.bs_shift_a = a, a + 4 * cv.cout
            cv.bs_mean_a, cv.bs_invstd_a = a + 8 * cv.cout, a + 12 * cv.cout
            a += 16 * cv.cout
            cv.bs_args = (bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                          bn.num_batches_tracked.data_ptr())
        self._bns = [cv.bn for cv in convs]
        self._bs_tensors = [t for m in self._bns for t in (m.running_mean, m.running_var, m.num_batches_tracked)]
        self._bs_cmax = max(cv.cout for cv in convs)

    def _bs_stats(self, cv, x_a, n):
        """Batch statistics of cv's raw output rows: scale / shift into cv's slot, the module's running buffers moved."""
        bn = cv.bn
        w_a, b_a, rm_a, rv_a, nbt_a = cv.bs_args
        rc = self._bs_stats_fn(x_a, n, cv.cout, w_a, b_a, bn.eps, -1.0 if bn.momentum is None else bn.momentum, rm_a, rv_a,
                               nbt_a, cv.bs_scale_a, cv.bs_shift_a, self._bs_ws_a, self._bs_ws_bytes, self._stream)
        if rc:
            C.check(rc, 'osb_bn_batch_stats')

    def _bs_apply(self, cv, x_a, n, relu=1, res_a=0, res_cv=None):
        """x = act(x * scale + shift + r) in place; r = res, or the raw downsample output `res_a` normalised with res_cv's slot."""
        rc = self._bs_apply_fn(x_a, n, cv.cout, cv.bs_scale_a, cv.bs_shift_a, res_a, res_cv.bs_scale_a if res_cv else 0,
                               res_cv.bs_shift_a if res_cv else 0, relu, self._stream)
        if rc:
            C.check(rc, 'osb_bn_apply_split')

    def _bs_norm(self, cv, x_a, n, relu=1, res_a=0, res_cv=None):
        self._bs_stats(cv, x_a, n)
        self._bs_apply(cv, x_a, n, relu, res_a, res_cv)
        return x_a

    # ---------------------------------------------------------------------------------------
    # Launch path: activations of one forward live in ONE arena tensor; layers are addressed by raw
    # device pointers and every convolution is a single ctypes call with prebuilt integer arguments
    # (no per-layer torch allocation, pointer boxing or workspace query: the Python dispatch cost per
    # layer has to stay below the ~20 us the coarse-level kernels take).
    def _plan_bytes(self, n):
        """Upper bound of split-row bytes for all activations of one forward (256-byte aligned slices)."""
        total = _al(n[0] * 4 * self.stem.cout)
        for l, (dconv, blocks) in enumerate(self.enc):
            total += _al(n[l + 1] * 4 * dconv.cout)
            for (c1, c2, ds) in blocks:
                total += _al(n[l + 1] * 4 * c1.cout) + _al(n[l + 1] * 4 * c2.cout) + (_al(n[l + 1] * 4 * ds.cout) if ds else 0)
        for j, (uconv, blocks) in enumerate(self.dec):
            l = 3 - j
            total += _al(n[l] * 4 * uconv.cout)
            for (c1, c2, ds) in blocks:
                total += _al(n[l] * 4 * c1.cout) + _al(n[l] * 4 * c2.cout) + (_al(n[l] * 4 * ds.cout) if ds else 0)
        return total

    def _chain_add(self, cv, s0, c0, s1, c1, nbr_a, n_rows, K, cout, res_a, relu, out_a, out_f32_a, row_map_a, cmap_a, cmap_cout,
                   independent=False):
        """Record one layer of the persistent chain.  Layers whose (row tile x N tile) count is at most `chain_max_tiles`
        share a launch with their neighbours (grid barrier between dependent layers); larger layers get their own launch.
        `independent`: the layer reads nothing the previous layer of the chain wrote (BasicBlock downsample next to conv1)."""
        ch = self._chain
        if self.layer_log is not None:
            self.layer_log.append((n_rows, K, c0 + c1, cout, 'dense-up' if cmap_a else ('res' if res_a else '')))
        tiles = -(-n_rows // 128) * max(1, -(-cout // 128))
        small = tiles <= self._chain_small
        if not (small and self._chain_prev_small):
            ch.cut()
        self._chain_prev_small = small
        ws_bytes = 0 if cmap_a else self._ws_query(n_rows, K, c0 + c1, cout)
        ws_a = 0
        if ws_bytes:
            self._ws_flip ^= 1                                   # consecutive split layers never share scratch
            ws_a = self._ws_a + self._ws_flip * (self._ws_bytes // 2)
            if ws_bytes > self._ws_bytes // 2:
                raise RuntimeError(f"FusedMinkUNet: split workspace of {ws_bytes} bytes exceeds the {self._ws_bytes // 2} provided")
        ch.add(s0, c0, s1, c1, nbr_a, n_rows, K, cv.wtiles_a, cout, cv.scale_a, cv.shift_a, res_a, relu, out_a, out_f32_a, row_map_a,
               cmap_a, cmap_cout, ws_a, ws_bytes, 0 if independent else 1)

    def _conv(self, cv, srcs, nbr_a, n_out, res_a=0, relu=1, out_f32_a=0, row_map_a=0, independent=False):
        """srcs: [(addr, channels, rows)] (one or two).  Returns the address of the split output (or 0)."""
        (s0, c0, r0) = srcs[0]
        (s1, c1, r1) = srcs[1] if len(srcs) > 1 else (0, 0, 0)
        out_a = 0
        if not out_f32_a:
            out_a = self._cursor
            self._cursor += _al(n_out * 4 * cv.cout)
        if self._chain_on:
            self._chain_add(cv, s0, c0, s1, c1, nbr_a, n_out, cv.K, cv.cout, res_a, relu, out_a, out_f32_a, row_map_a, 0, 0,
                            independent=independent)
            return out_a
        if self.layer_log is not None:
            self.layer_log.append((n_out, cv.K, c0 + c1, cv.cout, 'res' if res_a else ''))
        rc = self._fn(s0, c0, r0, s1, c1, r1, nbr_a, n_out, cv.K, cv.wpack_a, cv.cout, cv.scale_a, cv.shift_a, res_a, relu,
                      out_a, out_f32_a, row_map_a, self._ws_a, self._ws_bytes, self._flags, self._stream)
        if rc:
            C.check(rc, 'osb_conv_fwd_tc')
        return out_a

    def _chain_run(self):
        if self._chain_on:
            self._chain.run(self._flags, self._stream)

    def _stage(self, blocks, srcs, nbr3_a, n):
        if self.batch_stats:
            return self._stage_bs(blocks, srcs, nbr3_a, n)
        x = srcs
        for (c1, c2, ds) in blocks:
            y = self._conv(c1, x, nbr3_a, n)
            if ds is not None:
                r = self._conv(ds, x, 0, n, relu=0, independent=True)
            else:
                r = x[0][0]
            x = [(self._conv(c2, [(y, c1.cout, n)], nbr3_a, n, res_a=r), c2.cout, n)]
        return x[0]

    def _stage_bs(self, blocks, srcs, nbr3_a, n):
        """BasicBlocks with batch statistics: raw convolutions, each normalised in place; the downsample branch is only reduced
        (its normalisation happens inside conv2's apply pass, which reads it as the residual)."""
        x = srcs
        for (c1, c2, ds) in blocks:
            y = self._bs_norm(c1, self._conv(c1, x, nbr3_a, n, relu=0), n)
            if ds is not None:
                r = self._conv(ds, x, 0, n, relu=0)
                self._bs_stats(ds, r, n)
            else:
                r = x[0][0]
            z = self._conv(c2, [(y, c1.cout, n)], nbr3_a, n, relu=0)
            x = [(self._bs_norm(c2, z, n, res_a=r, res_cv=ds), c2.cout, n)]
        return x[0]

    def forward(self, coords, feats, coordinate_manager=None, head=None):
        """coords int32 [N,4] (batch,x,y,z), feats fp32 [N,cin], both CUDA, caller order.
        Returns fp32 [N, out_channels] in the caller's row order (== ``model(SparseTensor(feats, coords))``).
        batch_stats=True: == ``model(SparseTensor(feats, coords))`` in train mode, including the running-buffer updates."""
        return self._dp_forward(self._forward_no_grad, coords, feats, coordinate_manager, head)

    @torch.no_grad()
    def _forward_no_grad(self, coords, feats, coordinate_manager, head):
        if not self.batch_stats:
            return self._forward(coords, feats, coordinate_manager, head)
        if head is not None:
            raise NotImplementedError("FusedMinkUNet(batch_stats=True): the folded head is eval-only")
        if not self._net.training or not all(m.training for m in self._bns):
            self._check_mode()
        self._bs_started = False
        try:
            return self._forward(coords, feats, coordinate_manager, None)
        finally:
            if self._bs_started:
                # the kernels wrote the running buffers behind autograd's back: bump their versions as the module path's
                # in-place updates do, so that an eval-mode engine or fast_eval on this model re-folds them
                torch.autograd.graph.increment_version(self._bs_tensors)

    def _forward(self, coords, feats, coordinate_manager, head, tail=None):
        """The trunk, then the folded ``head``, the caller's ``tail(cur, n0, cm)`` on the last activation (split rows in
        internal order; its result is returned) or, with neither, the final layer."""
        C.require_cuda(feats, 'features')
        if self._sig != self._signature():                     # the source module changed since the weights were packed
            self.refresh()
        bs = self.batch_stats
        with torch.cuda.device(self.device):
            cm = coordinate_manager or CoordinateManager(coords, pyramid_levels=4 if self.use_pyramid else 0)
            self.last_cm = cm
            ts_list = [1]
            for _ in range(4):
                ts_list.append(cm.stride(ts_list[-1], 2))
            n = [cm.sets[t].n for t in ts_list]
            if bs:
                # level sizes are known here: refuse before anything is launched, so that no running buffer moves
                for l in range(5):
                    if n[l] < 2:
                        c = self.stem.cout if l == 0 else self.enc[l - 1][0].cout
                        raise ValueError(f"Expected more than 1 value per channel when training, got input size [{n[l]}, {c}] "
                                         f"(level {l}, tensor stride {ts_list[l]})")
                self._bs_started = True
            self._gen += 1
            nbr3 = [cm.kernel_map(t, t, 3).nbr for t in ts_list]
            down = [cm.kernel_map(ts_list[l], ts_list[l + 1], 2) for l in range(4)]
            up_nbr = [d.transposed().nbr for d in down] if not self.dense_up else None
            nbr3_a = [t.data_ptr() for t in nbr3]

            # Grow-only activation arena reused by every forward (activations never outlive one; the result is a separate
            # tensor).  Allocating ~1 GB per call made the caching allocator fragment against the 600 MB outputs and fall
            # back to cudaMalloc inside steps (10-120 ms stalls, 78 of them in 200 steps).
            need = self._plan_bytes(n) + 256
            if self._arena is None or self._arena.numel() < need:
                self._arena = None
                self._arena = torch.empty(int(need * 1.25), dtype=torch.uint8, device=self.device)
            self._cursor = _al(self._arena.data_ptr())
            if self._ws is None:
                self._ws = torch.empty(192 << 20, dtype=torch.uint8, device=self.device)      # two halves: consecutive split layers alternate
            self._ws_a, self._ws_bytes = self._ws.data_ptr(), self._ws.numel()
            self._stream = torch.cuda.current_stream().cuda_stream
            self._fn = C.lib().osb_conv_fwd_tc
            self._chain_on = self.use_chain and not bs           # batch statistics: one launch per layer (see module doc)
            if bs:
                # statistics workspace: grow-only like the arena; one suffices, the reductions run one after another in the stream
                ws_q = C.lib().osb_bn_stats_workspace_bytes
                need_bs = max(ws_q(nl, self._bs_cmax) for nl in n)
                if self._bs_ws is None or self._bs_ws.numel() < need_bs:
                    self._bs_ws = None
                    self._bs_ws = torch.empty(max(need_bs, 256), dtype=torch.uint8, device=self.device)
                self._bs_ws_a, self._bs_ws_bytes = self._bs_ws.data_ptr(), self._bs_ws.numel()
                self._bs_stats_fn, self._bs_apply_fn = C.lib().osb_bn_batch_stats, C.lib().osb_bn_apply_split
            if self._chain_on:
                if self._chain is None:
                    self._chain = tc.ConvChain(self.device, 160)
                    self._ws_query = C.lib().osb_conv_chain_workspace_bytes
                self._chain.begin()
                grid = C.lib().osb_conv_chain_grid()
                self._chain_small = self.chain_max_tiles if self.chain_max_tiles >= 0 else 2 * grid
                self._chain_prev_small = False
                self._ws_flip = 0
            # PDL: every kernel map / packed weight / BN constant is complete before the chain starts (maps are built
            # above, the stem kernel sits between them and the first convolution)
            self._flags = 1 if self.use_pdl else 0

            cs0 = cm.sets[1].ensure_lookup()
            f32 = feats.float().contiguous()
            x_int = torch.empty_like(f32)
            C.call('osb_gather_rows_f32', C.ptr(f32), C.ptr(cm.perm), n[0], f32.shape[1], C.ptr(x_int), C.stream_ptr())
            st = self.stem
            x_a = self._cursor
            self._cursor += _al(n[0] * 4 * st.cout)
            relu = 0 if bs else 1                           # batch statistics: raw convolutions (scale_a / shift_a are 0)
            if cs0.grid is not None:
                C.call('osb_conv_stem_fused_grid', C.ptr(x_int), st.cin, C.ptr(cs0.coords), n[0], C.ptr(cs0.grid), *cs0.grid_args,
                       st.ks, 1, C.ptr(st.w3), st.cout, st.scale_a, st.shift_a, relu, x_a, None, self._stream)
            else:
                C.call('osb_conv_stem_fused', C.ptr(x_int), st.cin, C.ptr(cs0.coords), n[0], C.ptr(cs0.slots), cs0.cap, st.ks, 1,
                       C.ptr(st.w3), st.cout, st.scale_a, st.shift_a, relu, x_a, None, self._stream)
            if bs:
                self._bs_norm(st, x_a, n[0])
            skips = [(x_a, st.cout, n[0])]
            cur = skips[0]
            for l, (dconv, blocks) in enumerate(self.enc):
                y = self._conv(dconv, [cur], down[l].nbr.data_ptr(), n[l + 1], relu=relu)
                if bs:
                    self._bs_norm(dconv, y, n[l + 1])
                cur = self._stage(blocks, [(y, dconv.cout, n[l + 1])], nbr3_a[l + 1], n[l + 1])
                skips.append(cur)
            for j, (uconv, blocks) in enumerate(self.dec):
                l = 3 - j                                   # output level of this transposed conv
                if self.dense_up and self._chain_on:
                    y = self._cursor
                    self._cursor += _al(n[l] * 4 * uconv.cout)
                    self._chain_add(uconv, cur[0], cur[1], 0, 0, 0, n[l + 1], 1, uconv.K * uconv.cout, 0, 1, y, 0, 0,
                                    down[l].nbr.data_ptr(), uconv.cout)
                elif self.dense_up:
                    y = self._cursor
                    self._cursor += _al(n[l] * 4 * uconv.cout)
                    if self.layer_log is not None:
                        self.layer_log.append((n[l + 1], 1, cur[1], uconv.K * uconv.cout, 'dense-up'))
                    rc = C.lib().osb_convtr_fwd_tc(cur[0], cur[1], n[l + 1], down[l].nbr.data_ptr(), uconv.K, uconv.wpack_a,
                                                   uconv.cout, uconv.scale_a, uconv.shift_a, relu, y, 0, self._flags, self._stream)
                    if rc:
                        C.check(rc, 'osb_convtr_fwd_tc')
                else:
                    y = self._conv(uconv, [cur], up_nbr[l].data_ptr(), n[l], relu=relu)
                if bs:
                    self._bs_norm(uconv, y, n[l])
                cur = self._stage(blocks, [(y, uconv.cout, n[l]), skips[l]], nbr3_a[l], n[l])
            if tail is not None:
                self._chain_run()
                return tail(cur, n[0], cm)
            if head is not None:                           # folded head: 96 -> (96 + K) conv, rows straight in caller order
                z = torch.empty((n[0], head.cout), dtype=torch.float32, device=self.device)
                self._conv(head, [cur], 0, n[0], relu=0, out_f32_a=z.data_ptr(), row_map_a=cm.perm.data_ptr())
                self._chain_run()
                return z
            fin = self.final
            out = torch.empty((n[0], fin.cout), dtype=torch.float32, device=self.device)
            if fin.wpack is not None:
                self._conv(fin, [cur], 0, n[0], relu=0, out_f32_a=out.data_ptr(), row_map_a=cm.perm.data_ptr())
                self._chain_run()
                return out
            self._chain_run()
            # odd head width (e.g. 20 classes): generic fp32 kernel, then restore the caller's order
            xf = torch.empty((n[0], cur[1]), dtype=torch.float32, device=self.device)
            C.call('osb_split_to_f32', cur[0], n[0], cur[1], C.ptr(xf), C.stream_ptr())
            C.call('osb_conv_fwd_f32', C.ptr(xf), fin.cin, None, n[0], 1, C.ptr(fin.w3), fin.cin, fin.cout, 0, C.ptr(out),
                   C.stream_ptr())
            ext = torch.empty_like(out)
            C.call('osb_gather_rows_f32', C.ptr(out), C.ptr(cm.inv_perm), n[0], fin.cout, C.ptr(ext), C.stream_ptr())
            return ext

    __call__ = forward

    def forward_train(self, coords, feats, rows=None):
        """Training forward of a batch_stats engine with a device backward (openscene_b200/engine_train.py).
        Returns fp32 rows with a grad_fn: ``model(SparseTensor(feats, coords))`` (rows=None, caller order) or its ``[rows]``
        (bool mask or int64 caller-row index; only those rows go through the final 1x1x1 layer).  ``loss.backward()`` then
        writes / accumulates ``.grad`` of every parameter of the model.  The running buffers move once per call."""
        from . import engine_train
        return self._dp_forward(engine_train.forward_train, self, coords, feats, rows)

    def forward_train_ce(self, coords, feats, labels, ignore_index=-100):
        """Training step of a per-voxel classifier on a batch_stats engine (run/train_mink.py): returns ``(loss, pred)`` with
        ``loss == F.cross_entropy(model(SparseTensor(feats, coords)), labels, ignore_index=ignore_index)`` (0-dim fp32 with a
        grad_fn) and ``pred == output.max(1)[1]`` (int64 [N], caller order, up to ties).  Any head of 1 to 160 classes on a
        trunk of width a multiple of 32 up to 384.  ``loss.backward()`` fills ``.grad`` of every parameter; the logits are
        never materialised (openscene_b200/engine_train.py, csrc/ce_head.cu)."""
        from . import engine_train
        return self._dp_forward(engine_train.forward_train_ce, self, coords, feats, labels, ignore_index)

    def forward_train_cosine(self, coords, feats, feat_3d, rows):
        """Distillation step with run/distill.py's cosine loss on a batch_stats engine: returns the 0-dim fp32 loss
        ``distill_loss(forward_train(coords, feats, rows), feat_3d)`` with a grad_fn, where ``rows`` is the bool mask or int64
        caller-row index of the supervised rows and ``feat_3d`` their fp16 [M, C] targets in that order.  A head of 512 or 768
        channels on a trunk of width a multiple of 32 up to 384; ``loss.backward()`` fills ``.grad`` of every parameter.  The
        [M, C] rows and their gradient are never materialised (openscene_b200/engine_train.py, csrc/cos_head.cu)."""
        from . import engine_train
        return self._dp_forward(engine_train.forward_train_cosine, self, coords, feats, feat_3d, rows)

    def forward_train_l1(self, coords, feats, feat_3d, rows):
        """Distillation step with run/distill.py's L1 loss on a batch_stats engine: returns the 0-dim fp32 loss
        ``distill_loss(forward_train(coords, feats, rows), feat_3d, 'l1')`` with a grad_fn; arguments and supported heads as
        in forward_train_cosine.  The [M, C] rows and their gradient are never materialised; the backward reads the 2-bit
        signs of f - t the forward kept (openscene_b200/engine_train.py, csrc/l1_head.cu)."""
        from . import engine_train
        return self._dp_forward(engine_train.forward_train_l1, self, coords, feats, feat_3d, rows)

    @torch.no_grad()
    def forward_eval_ce(self, coords, feats, labels, inds_reverse, loss, areas, bad, ignore_index=255, pred=None):
        """Validation tail of a per-voxel classifier on the eval engine (run/train_mink.py's validate() after
        ``output = model(sinput)``): the trunk runs as in ``forward``, and one launch (osb_ce_head_eval) replaces the final
        layer, the ``output[inds_reverse]`` gather, ``CrossEntropyLoss(ignore_index)``, ``output.max(1)[1]`` and
        ``intersectionAndUnionGPU``; the logits are never written.  No host synchronisation.

        labels: int32 / int64 [n_pts] per point; inds_reverse: int64 [n_pts] voxel (caller row) of every point, or None (one
        point per row).  Outputs, device tensors the caller owns: ``loss`` fp32 (first element) = the loss over points with
        a label in [0, C) (NaN when there is none), ``areas`` int64 [3, C] += intersection | output | target counts, ``bad``
        int32 (first element) += points whose label is outside [0, C) and not ``ignore_index`` (left out of the loss and the
        counts), ``pred`` (optional) int64 [n_pts] = the first argmax per point."""
        from .engine_train import CE_CIN, CE_MAX_CLASSES
        if self.batch_stats:
            raise NotImplementedError("forward_eval_ce: an eval-mode engine (FusedMinkUNet without batch_stats) folds BatchNorm "
                                      "into the trunk; validate on FusedMinkUNet(model.eval())")
        fin = self.final
        if fin.cout > CE_MAX_CLASSES or fin.cin not in CE_CIN or fin.K != 1:
            raise NotImplementedError(f"forward_eval_ce: a 1x1x1 head of {fin.cin} -> {fin.cout} channels (supported: input "
                                      f"width a multiple of 32 up to 384, 1 to {CE_MAX_CLASSES} classes)")
        dev = self.device
        n_rows = feats.shape[0]
        inv = None if inds_reverse is None else inds_reverse.to(dev, torch.int64, non_blocking=True).contiguous().view(-1)
        n_pts = n_rows if inv is None else inv.numel()
        lab = torch.as_tensor(labels).to(dev, non_blocking=True).contiguous().view(-1)
        if lab.dtype not in (torch.int32, torch.int64):
            lab = lab.long()
        if lab.numel() != n_pts:
            raise ValueError(f"forward_eval_ce: {lab.numel()} labels for {n_pts} points")
        for t, what, dt, k in ((loss, 'loss', torch.float32, 1), (areas, 'areas', torch.int64, 3 * fin.cout),
                               (bad, 'bad', torch.int32, 1), (pred, 'pred', torch.int64, n_pts)):
            if t is None and what == 'pred':
                continue
            if t.device != dev or t.dtype != dt or not t.is_contiguous() or t.numel() < k:
                raise ValueError(f"forward_eval_ce: {what} must be a contiguous {dt} tensor of at least {k} elements on {dev}")

        def tail(cur, n0, cm):
            fin = self.final                                # _forward re-packs (a new final) when the weights changed
            need = C.lib().osb_ce_head_eval_workspace_bytes(n_pts, cur[1], fin.cout)
            if self._ce_ws is None or self._ce_ws.numel() < need:
                self._ce_ws = None
                self._ce_ws = torch.empty(max(need, 256), dtype=torch.uint8, device=dev)
            rc = C.lib().osb_ce_head_eval(cur[0], n0, cur[1], fin.w3.data_ptr(), fin.cout, cm.inv_perm.data_ptr(),
                                          C.ptr(inv), n_pts, lab.data_ptr(), int(lab.dtype == torch.int64), int(ignore_index),
                                          C.ptr(pred), loss.data_ptr(), areas.data_ptr(), bad.data_ptr(), self._ce_ws.data_ptr(),
                                          self._ce_ws.numel(), self._stream)
            if rc:
                C.check(rc, 'osb_ce_head_eval')
        self._forward(coords, feats, None, None, tail)

    # ---------------------------------------------------------------------------------------
    def fold_head(self, text_features):
        """Pre-compute the folded head for a set of unit-norm text embeddings [K, C_out]:
        W W^T = L L^T (Cholesky, fp64) and U = W T^T, packed as one 1x1x1 convolution 96 -> (96 + K)."""
        if self.batch_stats:
            raise NotImplementedError("fold_head: the folded head is eval-only (FusedMinkUNet without batch_stats)")
        W = self.final.w3[0].double()                                    # [cin, cout]
        T = text_features.to(W.device).double()                          # [K, cout]
        G = W @ W.t()
        G = G + 1e-12 * torch.eye(G.shape[0], device=G.device, dtype=G.dtype) * G.diagonal().mean()
        L = torch.linalg.cholesky(G)                                     # x G x^T = |x L|^2
        U = W @ T.t()
        cin, k = W.shape[0], T.shape[0]
        cout = ((cin + k + 31) // 32) * 32
        w = torch.zeros((1, cin, cout), dtype=torch.float32, device=W.device)
        w[0, :, :cin] = L.float()
        w[0, :, cin:cin + k] = U.float()
        cv = _Conv.__new__(_Conv)
        cv.K, cv.cin, cv.cout, cv.ks, cv.stride, cv.transpose = 1, cin, cout, 1, 1, False
        cv.w3, cv.wpack = w, tc.pack_weights(w)
        cv.wtiles = tc.pack_weight_tiles(w)
        cv.scale = cv.shift = None
        cv.wpack_a, cv.wtiles_a, cv.scale_a, cv.shift_a = cv.wpack.data_ptr(), cv.wtiles.data_ptr(), 0, 0
        cv.n_ntiles = max(1, -(-cout // 128))
        return (cv, cin, k, self._signature())               # the signature lets forward_scores refuse a head folded from older weights

    @torch.no_grad()
    def forward_scores(self, coords, feats, folded, want_scores=True):
        """Cosine scores / labels of every voxel against the folded text set (``fold_head``), equal to
        ``match(normalize(forward(coords, feats)), text)`` up to rounding, without the 768-d features.
        Returns (scores fp16 [N,K] or None, label int64 [N], smax fp32 [N]) in the caller's row order."""
        if self.batch_stats:
            raise NotImplementedError("forward_scores: the folded head is eval-only (FusedMinkUNet without batch_stats)")
        cv, cin, k = folded[:3]
        if len(folded) > 3 and folded[3] != self._signature():
            raise RuntimeError("forward_scores: the folded head was built from weights that have changed since; call fold_head again")
        z = self.forward(coords, feats, head=cv)
        n = z.shape[0]
        scores = torch.empty((n, k), dtype=torch.float16, device=self.device) if want_scores else None
        label = torch.empty(n, dtype=torch.int64, device=self.device)
        smax = torch.empty(n, dtype=torch.float32, device=self.device)
        C.call('osb_folded_head_finish', C.ptr(z), n, cv.cout, cin, k, C.ptr(scores), C.ptr(label), C.ptr(smax), C.stream_ptr())
        return scores, label, smax

    def conv_census(self, cm):
        """Per-convolution (name, pairs, cin, cout, n_in, n_out) of the last forward: algorithmic flops / bytes
        (SURVEY.md 8d definitions) for bench.py's roofline accounting."""
        ts = [1, 2, 4, 8, 16]
        n = [cm.sets[t].n for t in ts]
        p3 = [cm.kernel_map(t, t, 3).num_pairs() for t in ts]
        rows = []
        k5 = cm.kmaps.get((1, 1, 5, 1))
        rows.append(('stem', k5.num_pairs() if k5 is not None else None, self.stem.cin, self.stem.cout, n[0], n[0], 125))

        def stage(tag, blocks, l, cin_first):
            for bi, (c1, c2, ds) in enumerate(blocks):
                rows.append((f'{tag}.{bi}.conv1', p3[l], c1.cin, c1.cout, n[l], n[l], 27))
                rows.append((f'{tag}.{bi}.conv2', p3[l], c2.cin, c2.cout, n[l], n[l], 27))
                if ds is not None:
                    rows.append((f'{tag}.{bi}.downsample', n[l], ds.cin, ds.cout, n[l], n[l], 1))
        for l, (dconv, blocks) in enumerate(self.enc):
            rows.append((f'down{l + 1}', n[l], dconv.cin, dconv.cout, n[l], n[l + 1], 8))
            stage(f'block{l + 1}', blocks, l + 1, dconv.cout)
        for j, (uconv, blocks) in enumerate(self.dec):
            l = 3 - j
            rows.append((f'up{j + 4}', n[l], uconv.cin, uconv.cout, n[l + 1], n[l], 8))
            stage(f'block{j + 5}', blocks, l, None)
        rows.append(('final', n[0], self.final.cin, self.final.cout, n[0], n[0], 1))
        return rows
