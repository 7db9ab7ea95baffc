"""Training step of the fused MinkUNet engine: ``FusedMinkUNet.forward_train`` and its device backward.

Forward: the launch sequence of ``FusedMinkUNet(model, batch_stats=True)`` on the per-layer path, except that every BatchNorm
keeps its raw convolution output ``z`` (``osb_bn_batch_stats_save`` also writes the batch mean / invstd, and
``osb_bn_apply_split_out`` writes the normalised rows ``y`` to a separate buffer).  The final 1x1x1 layer runs on the selected
rows only: ``osb_conv_fwd_tc`` with K = 1 and a map listing their internal rows.

Backward, in reverse layer order, everything in split rows:
  * BatchNorm (+ ReLU + residual): ``osb_bn_backward_reduce`` (affine gradients) and ``osb_bn_backward_apply`` (dz; for an
    identity shortcut also the masked gradient g' the block input receives); the downsample branch's BatchNorm reads the same
    masked gradient through the block output's ReLU mask;
  * convolutions: wgrad ``osb_conv_wgrad_tc`` (forward map), dgrad ``osb_conv_fwd_tc`` with W^T packed over the map with the
    roles swapped (stride 2: the transposed down map; dense transposed convolutions: the down map itself).  A convolution that
    reads ``[up | skip]`` runs one wgrad and one dgrad per source;
  * the stem: wgrad only, ``osb_conv_wgrad_tc`` over the 5^3 map with the 3 input channels zero-padded to 32 (the input
    features get no gradient).
A tensor with several consumers collects its gradient in a fixed order through the ``res`` operand of the dgrad (output and
residual never alias), so two identical steps give bit-identical gradients.

``forward_train_ce`` (per-voxel classification, run/train_mink.py) runs the same trunk and replaces the final layer by
``osb_ce_head_fwd`` (head product, log-sum-exp, NLL over the labelled rows, argmax in caller order); its backward starts with
``osb_ce_head_bwd``, which writes the head's weight gradient and the trunk output's gradient, and continues as above.
``forward_train_cosine`` (distillation with run/distill.py's cosine loss) does the same with ``osb_cos_head_fwd`` (head product
and cosine loss on the selected rows) and ``osb_cos_head_bwd``: the C-wide rows and their gradient never exist.
``forward_train_l1`` (the L1 loss) does the same with ``osb_l1_head_fwd`` (head product, L1 loss and the packed signs of
f - t) and ``osb_l1_head_bwd`` (the gradients from the signs alone).

With a process group (``FusedMinkUNet(model, batch_stats=True, process_group=pg)``) the backward all-reduces the gradients as
DistributedDataParallel does: the flat gradient buffer is cut at parameter boundaries into buckets, from the end of the
parameter list (the head's and decoder's gradients are written first), of about 1 MiB for the first and 25 MiB for the others.
Right after the tape item that writes a bucket's last slot, the bucket is divided by the world size and all-reduced
asynchronously, ordered behind the launches already on the current stream; the backward waits on every collective (a
stream wait for NCCL) before it returns, so the optimiser and the next forward read reduced gradients and no collective
overlaps the next forward's launches."""
import torch
import torch.distributed as dist
from torch.autograd.function import once_differentiable

from . import _cabi as C
from . import tc
from .coords import CoordinateManager

_GCHUNK = 64 << 20
_FIRST_BUCKET_BYTES = 1 << 20                     # torch.distributed._DEFAULT_FIRST_BUCKET_BYTES
_BUCKET_BYTES = 25 << 20                          # DistributedDataParallel's bucket_cap_mb=25


def _al(x):
    return (x + 255) & ~255


def plan_train_bytes(eng, n):
    """Activation bytes of one forward_train: raw and normalised rows of every BatchNorm layer (downsample: raw only)."""
    total = 2 * _al(n[0] * 4 * eng.stem.cout)
    for l, (dconv, blocks) in enumerate(eng.enc):
        total += 2 * _al(n[l + 1] * 4 * dconv.cout)
        for (c1, c2, ds) in blocks:
            total += 2 * _al(n[l + 1] * 4 * c1.cout) + 2 * _al(n[l + 1] * 4 * c2.cout) + (_al(n[l + 1] * 4 * ds.cout) if ds else 0)
    for j, (uconv, blocks) in enumerate(eng.dec):
        l = 3 - j
        total += 2 * _al(n[l] * 4 * uconv.cout)
        for (c1, c2, ds) in blocks:
            total += 2 * _al(n[l] * 4 * c1.cout) + 2 * _al(n[l] * 4 * c2.cout) + (_al(n[l] * 4 * ds.cout) if ds else 0)
    return total


class _Node:
    """One convolution (+ BatchNorm) of the forward: what its backward reads."""
    __slots__ = ('cv', 'z', 'y', 'n', 'srcs', 'K', 'nbr_f', 'nbr_b', 'n_out', 'stem')

    def __init__(self, cv, z, y, n, srcs, K, nbr_f, nbr_b, stem=False):
        self.cv, self.z, self.y, self.n, self.srcs, self.K, self.nbr_f, self.nbr_b = cv, z, y, n, srcs, K, nbr_f, nbr_b
        self.n_out, self.stem = n, stem


class _Graph:
    pass


def _refuse(eng, feats):
    if not eng.batch_stats:
        raise RuntimeError("forward_train: build the engine with FusedMinkUNet(model, batch_stats=True) from a train-mode model")
    eng._check_mode()
    if feats.requires_grad:
        raise NotImplementedError("forward_train: the gradient of the input features is not computed (feats.requires_grad)")


def forward_train(eng, coords, feats, rows=None):
    _refuse(eng, feats)
    C.require_cuda(feats, 'features')
    if eng._sig != eng._signature():                     # weights changed (optimiser step): re-pack before anything runs
        eng.refresh()
    if eng.final.wpack is None:
        raise NotImplementedError("forward_train: the final layer's widths must be multiples of 32 (tensor-core head); "
                                  "a classifier head with cross-entropy trains through forward_train_ce")
    _ensure_bwd_packs(eng)
    params = list(eng._net.parameters())
    return _TrainFunction.apply(eng, coords, feats, rows, *params)


CE_MAX_CLASSES = 160
CE_CIN = (32, 64, 96, 128, 160, 192, 224, 256, 288, 320, 352, 384)


def forward_train_ce(eng, coords, feats, labels, ignore_index=-100):
    """(loss, pred): ``F.cross_entropy(model(SparseTensor(feats, coords)), labels, ignore_index=ignore_index)`` with a grad_fn,
    and ``output.max(1)[1]`` (int64, caller order).  The trunk runs as in forward_train; the final 1x1x1 layer, the loss and
    the argmax are one launch (osb_ce_head_fwd) and its backward another (osb_ce_head_bwd): the logits never exist."""
    _refuse(eng, feats)
    C.require_cuda(feats, 'features')
    if not isinstance(labels, torch.Tensor) or labels.dtype == torch.bool or labels.is_floating_point() or labels.is_complex():
        raise TypeError(f"forward_train_ce: labels must be an integer tensor (got {getattr(labels, 'dtype', type(labels))})")
    if labels.dim() != 1 or labels.shape[0] != feats.shape[0]:
        raise ValueError(f"forward_train_ce: labels of shape {tuple(labels.shape)} for {feats.shape[0]} rows (expected [N])")
    if eng._sig != eng._signature():
        eng.refresh()
    fin = eng.final
    if fin.cout > CE_MAX_CLASSES or fin.cin not in CE_CIN or fin.K != 1:
        raise NotImplementedError(f"forward_train_ce: a 1x1x1 head of {fin.cin} -> {fin.cout} channels (supported: input width a "
                                  f"multiple of 32 up to 384, 1 to {CE_MAX_CLASSES} classes)")
    labels = labels.to(eng.device)
    if labels.dtype not in (torch.int32, torch.int64):
        labels = labels.long()
    labels = labels.contiguous()
    ignore_index = int(ignore_index)
    bad = (labels != ignore_index) & ((labels < 0) | (labels >= fin.cout))
    if bool(bad.any()):                                 # before anything is launched: no running buffer moves
        raise IndexError(f"forward_train_ce: Target {int(labels[bad][0])} is out of bounds for {fin.cout} classes")
    _ensure_bwd_packs(eng)
    params = list(eng._net.parameters())
    return _CEFunction.apply(eng, coords, feats, labels, ignore_index, *params)


def _ce_workspace(eng, n, cin, c, query='osb_ce_head_workspace_bytes'):
    """the engine's head workspace (shared by the cross-entropy, cosine and L1 heads), grown to the query's size"""
    need = getattr(C.lib(), query)(n, cin, c)
    if eng._ce_ws is None or eng._ce_ws.numel() < need:
        eng._ce_ws = None
        eng._ce_ws = torch.empty(max(need, 256), dtype=torch.uint8, device=eng.device)
    return eng._ce_ws.data_ptr(), eng._ce_ws.numel()


def _ce_forward(eng, cm, cur, n0, ce, tape):
    """osb_ce_head_fwd on the trunk's last activation; records what the backward reads"""
    labels, ignore = ce
    fin, dev = eng.final, eng.device
    lse = torch.empty(n0, dtype=torch.float32, device=dev)
    pred = torch.empty(n0, dtype=torch.int64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    n_valid = torch.empty(1, dtype=torch.int64, device=dev)
    ws_a, ws_b = _ce_workspace(eng, n0, cur[1], fin.cout)
    i64 = 1 if labels.dtype == torch.int64 else 0
    rc = C.lib().osb_ce_head_fwd(cur[0], n0, cur[1], fin.w3.data_ptr(), fin.cout, cm.perm.data_ptr(), labels.data_ptr(), i64,
                                 ignore, lse.data_ptr(), pred.data_ptr(), loss.data_ptr(), n_valid.data_ptr(), ws_a, ws_b,
                                 eng._stream)
    if rc:
        C.check(rc, 'osb_ce_head_fwd')
    tape.append(('ce_head', (_Node(fin, 0, 0, n0, [cur], 1, 0, 0), cm.perm, labels, ignore, lse, n_valid)))
    return loss, pred


def _ce_backward(eng, item, g, slot, galloc, grads, stream):
    """osb_ce_head_bwd: dW into the final kernel's gradient slot, dx = the gradient of the trunk's last activation"""
    nd, perm, labels, ignore, lse, n_valid = item
    cv = nd.cv
    (src, c, n0), = nd.srcs
    dx = galloc(n0 * 4 * c)
    ws_a, ws_b = _ce_workspace(eng, n0, c, cv.cout)
    i64 = 1 if labels.dtype == torch.int64 else 0
    rc = C.lib().osb_ce_head_bwd(src, n0, c, cv.w3.data_ptr(), cv.cout, perm.data_ptr(), labels.data_ptr(), i64, ignore,
                                 lse.data_ptr(), g.data_ptr(), n_valid.data_ptr(), dx, slot(cv.mod.kernel).data_ptr(), ws_a, ws_b,
                                 stream)
    if rc:
        C.check(rc, 'osb_ce_head_bwd')
    grads[src] = dx


class _CEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng, coords, feats, labels, ignore, *params):
        graph = _run_forward(eng, coords, feats, None, ce=(labels, ignore))
        loss, pred = graph.out
        graph.out = None
        ctx.eng, ctx.graph = eng, graph
        ctx.save_for_backward(*params)
        ctx.mark_non_differentiable(pred)
        return loss, pred

    @staticmethod
    @once_differentiable
    def backward(ctx, g, _g_pred):
        params = ctx.saved_tensors
        grads = _run_backward(ctx.eng, ctx.graph, g, params)
        ctx.graph = None
        return (None, None, None, None, None) + tuple(grads)


COS_WIDTHS = (512, 768)


def forward_train_cosine(eng, coords, feats, feat_3d, rows):
    """0-dim fp32 loss with a grad_fn: ``distill_loss(forward_train(coords, feats, rows), feat_3d)`` with the cosine loss.
    The trunk runs as in forward_train; the final 1x1x1 layer and the loss are one launch (osb_cos_head_fwd) and their
    backward another (osb_cos_head_bwd): the [M, C] rows and their gradient never exist.  feat_3d: fp16 [M, C] on the
    engine's device, in the order of ``rows`` (bool mask or int64 caller-row index, as in forward_train)."""
    _refuse_distill_head(eng, feats, feat_3d, rows, 'forward_train_cosine')
    params = list(eng._net.parameters())
    return _CosFunction.apply(eng, coords, feats, rows, feat_3d.contiguous(), *params)


def _refuse_distill_head(eng, feats, feat_3d, rows, what):
    """everything the device distillation heads refuse, before anything is launched; re-packs a stale engine"""
    _refuse(eng, feats)
    C.require_cuda(feats, 'features')
    if eng._sig != eng._signature():
        eng.refresh()
    fin = eng.final
    if fin.cout not in COS_WIDTHS or fin.cin not in CE_CIN or fin.K != 1:
        raise NotImplementedError(f"{what}: a 1x1x1 head of {fin.cin} -> {fin.cout} channels (supported: input "
                                  f"width a multiple of 32 up to 384, output width 512 or 768); train it with forward_train "
                                  f"and distill_loss")
    if not isinstance(feat_3d, torch.Tensor) or feat_3d.dtype != torch.float16:
        raise TypeError(f"{what}: feat_3d must be an fp16 tensor (got {getattr(feat_3d, 'dtype', type(feat_3d))})")
    if feat_3d.dim() != 2 or feat_3d.shape[1] != fin.cout:
        raise ValueError(f"{what}: feat_3d of shape {tuple(feat_3d.shape)} for a head of {fin.cout} channels "
                         f"(expected [M, {fin.cout}])")
    if feat_3d.device != eng.device:
        raise ValueError(f"{what}: feat_3d is on {feat_3d.device}, the engine on {eng.device}")
    if rows is None:
        raise ValueError(f"{what}: rows (the supervised rows) is required")
    _ensure_bwd_packs(eng)


def _cos_forward(eng, cur, n0, sel, target, tape):
    """osb_cos_head_fwd on the trunk's last activation; records what the backward reads"""
    fin, dev = eng.final, eng.device
    m = sel.shape[0]
    state = torch.empty((m, 3), dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    ws_a, ws_b = _ce_workspace(eng, m, cur[1], fin.cout, 'osb_cos_head_workspace_bytes')
    rc = C.lib().osb_cos_head_fwd(cur[0], n0, cur[1], fin.w3.data_ptr(), fin.cout, sel.data_ptr(), m, target.data_ptr(),
                                  state.data_ptr(), loss.data_ptr(), ws_a, ws_b, eng._stream)
    if rc:
        C.check(rc, 'osb_cos_head_fwd')
    tape.append(('cos_head', (_Node(fin, 0, 0, n0, [cur], 1, 0, 0), sel, target, state)))
    return loss


def _cos_backward(eng, item, g, slot, galloc, grads, stream):
    """osb_cos_head_bwd: dW into the final kernel's gradient slot, dx = the gradient of the trunk's last activation"""
    nd, sel, target, state = item
    cv = nd.cv
    (src, c, n0), = nd.srcs
    m = sel.shape[0]
    dx = galloc(n0 * 4 * c)
    ws_a, ws_b = _ce_workspace(eng, m, c, cv.cout, 'osb_cos_head_workspace_bytes')
    rc = C.lib().osb_cos_head_bwd(src, n0, c, cv.w3.data_ptr(), cv.cout, sel.data_ptr(), m, target.data_ptr(), state.data_ptr(),
                                  g.data_ptr(), dx, slot(cv.mod.kernel).data_ptr(), ws_a, ws_b, stream)
    if rc:
        C.check(rc, 'osb_cos_head_bwd')
    grads[src] = dx


class _CosFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng, coords, feats, rows, target, *params):
        graph = _run_forward(eng, coords, feats, rows, cos=target)
        loss = graph.out
        graph.out = None
        ctx.eng, ctx.graph = eng, graph
        ctx.save_for_backward(*params)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        params = ctx.saved_tensors
        grads = _run_backward(ctx.eng, ctx.graph, g, params)
        ctx.graph = None
        return (None, None, None, None, None) + tuple(grads)


def forward_train_l1(eng, coords, feats, feat_3d, rows):
    """0-dim fp32 loss with a grad_fn: ``distill_loss(forward_train(coords, feats, rows), feat_3d, 'l1')``, the mean of
    |f - t| over the [M, C] elements.  The trunk runs as in forward_train; the final 1x1x1 layer and the loss are one launch
    sequence (osb_l1_head_fwd, which keeps the 2-bit sign of every f - t) and their backward another (osb_l1_head_bwd, from
    the signs alone): the [M, C] rows and their gradient never exist.  feat_3d and rows as in forward_train_cosine."""
    _refuse_distill_head(eng, feats, feat_3d, rows, 'forward_train_l1')
    params = list(eng._net.parameters())
    return _L1Function.apply(eng, coords, feats, rows, feat_3d.contiguous(), *params)


def _l1_forward(eng, cur, n0, sel, target, tape):
    """osb_l1_head_fwd on the trunk's last activation; records the signs the backward reads"""
    fin, dev = eng.final, eng.device
    m = sel.shape[0]
    signs = torch.empty((m, fin.cout // 16), dtype=torch.int32, device=dev)      # uint32 words (torch has no uint32 kernels)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    ws_a, ws_b = _ce_workspace(eng, m, cur[1], fin.cout, 'osb_l1_head_workspace_bytes')
    rc = C.lib().osb_l1_head_fwd(cur[0], n0, cur[1], fin.w3.data_ptr(), fin.cout, sel.data_ptr(), m, target.data_ptr(),
                                 signs.data_ptr(), loss.data_ptr(), ws_a, ws_b, eng._stream)
    if rc:
        C.check(rc, 'osb_l1_head_fwd')
    tape.append(('l1_head', (_Node(fin, 0, 0, n0, [cur], 1, 0, 0), sel, signs)))
    return loss


def _l1_backward(eng, item, g, slot, galloc, grads, stream):
    """osb_l1_head_bwd: dW into the final kernel's gradient slot, dx = the gradient of the trunk's last activation"""
    nd, sel, signs = item
    cv = nd.cv
    (src, c, n0), = nd.srcs
    m = sel.shape[0]
    dx = galloc(n0 * 4 * c)
    ws_a, ws_b = _ce_workspace(eng, m, c, cv.cout, 'osb_l1_head_workspace_bytes')
    rc = C.lib().osb_l1_head_bwd(src, n0, c, cv.w3.data_ptr(), cv.cout, sel.data_ptr(), m, signs.data_ptr(), g.data_ptr(), dx,
                                 slot(cv.mod.kernel).data_ptr(), ws_a, ws_b, stream)
    if rc:
        C.check(rc, 'osb_l1_head_bwd')
    grads[src] = dx


class _L1Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng, coords, feats, rows, target, *params):
        graph = _run_forward(eng, coords, feats, rows, l1=target)
        loss = graph.out
        graph.out = None
        ctx.eng, ctx.graph = eng, graph
        ctx.save_for_backward(*params)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        params = ctx.saved_tensors
        grads = _run_backward(ctx.eng, ctx.graph, g, params)
        ctx.graph = None
        return (None, None, None, None, None) + tuple(grads)


def _ensure_bwd_packs(eng):
    """W^T of every convolution, per source for the ones reading [up | skip] (dgrad operands); built once per re-pack."""
    convs = [cv for (c0, blocks) in eng.enc + eng.dec for cv in [c0] + [x for blk in blocks for x in blk if x is not None]]
    convs.append(eng.final)
    with torch.cuda.device(eng.device), torch.no_grad():
        for cv in convs:
            if cv.bwd is None:
                w3 = cv.mod.kernel.detach()
                w3 = w3.unsqueeze(0) if w3.dim() == 2 else w3
                cv.bwd = w3                                              # split per source on first use (_packs_for)
    eng._bwd_convs = convs


def _packs_for(cv, widths):
    """[(lo, hi, W[:, lo:hi, :]^T packed)] for the given source widths (memoised on the _Conv)."""
    if isinstance(cv.bwd, list):
        return cv.bwd
    w3, out, lo = cv.bwd, [], 0
    for c in widths:
        out.append((lo, lo + c, tc.pack_weights(w3[:, lo:lo + c, :], transpose_w=True)))
        lo += c
    cv.bwd = out
    return out


def _select(cm, rows, n0, dev):
    """int32 internal rows of the selected caller rows (output order), or refuse."""
    if rows is None:
        return cm.inv_perm
    if rows.dtype == torch.bool:
        if rows.shape != (n0,):
            raise ValueError(f"forward_train: mask of shape {tuple(rows.shape)} for {n0} rows")
        idx = rows.to(dev).nonzero().squeeze(1)
    elif rows.dtype in (torch.int64, torch.int32):
        idx = rows.to(dev).long().reshape(-1)
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= n0):
            raise IndexError(f"forward_train: row index out of range for {n0} rows")
        if torch.unique(idx).numel() != idx.numel():
            raise ValueError("forward_train: repeated row indices are not supported (the head's dgrad scatters one row each)")
    else:
        raise TypeError("forward_train: rows must be None, a bool mask or an int64 index")
    if idx.numel() == 0:
        raise ValueError("forward_train: no rows selected")
    return cm.inv_perm[idx].to(torch.int32).contiguous()


class _TrainFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng, coords, feats, rows, *params):
        graph = _run_forward(eng, coords, feats, rows)
        ctx.eng, ctx.graph = eng, graph
        ctx.save_for_backward(*params)
        return graph.out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        params = ctx.saved_tensors                      # raises torch's version error if a weight changed in place since
        grads = _run_backward(ctx.eng, ctx.graph, g, params)
        ctx.graph = None
        return (None, None, None, None) + tuple(grads)


def _run_forward(eng, coords, feats, rows, ce=None, cos=None, l1=None):
    dev = eng.device
    st = eng.stem
    with torch.cuda.device(dev):
        cm = CoordinateManager(coords, pyramid_levels=4 if eng.use_pyramid else 0)
        ts = [1]
        for _ in range(4):
            ts.append(cm.stride(ts[-1], 2))
        n = [cm.sets[t].n for t in ts]
        for l in range(5):
            if n[l] < 2:
                c = st.cout if l == 0 else eng.enc[l - 1][0].cout
                raise ValueError(f"Expected more than 1 value per channel when training, got input size [{n[l]}, {c}] "
                                 f"(level {l}, tensor stride {ts[l]})")
        sel = _select(cm, rows, n[0], dev) if ce is None else None
        for what, tgt in (('forward_train_cosine', cos), ('forward_train_l1', l1)):
            if tgt is not None and tgt.shape[0] != sel.shape[0]:
                raise ValueError(f"{what}: feat_3d has {tgt.shape[0]} rows for {sel.shape[0]} selected rows")
        eng._gen += 1                                    # from here on the arena is overwritten
        eng.last_cm = cm
        m3 = [cm.kernel_map(t, t, 3) for t in ts]
        down = [cm.kernel_map(ts[l], ts[l + 1], 2) for l in range(4)]
        # every map the backward reads is built now, before the first launch of the step
        nbr3 = [(k.nbr.data_ptr(), k.transposed().nbr.data_ptr()) for k in m3]
        dn = [(d.nbr.data_ptr(), d.transposed().nbr.data_ptr()) for d in down]
        m, sel_t = n[0], None
        if ce is None:
            m = sel.shape[0]
        if ce is None and cos is None and l1 is None:
            sel_t = torch.empty(n[0], dtype=torch.int32, device=dev)
            C.call('osb_kernel_map_transpose', C.ptr(sel), m, 1, C.ptr(sel_t), n[0], C.stream_ptr())
        k5 = cm.kernel_map(1, 1, st.ks)

        need = plan_train_bytes(eng, n) + 256
        if eng._arena is None or eng._arena.numel() < need:
            eng._arena = None
            eng._arena = torch.empty(int(need * 1.25), dtype=torch.uint8, device=dev)
        eng._cursor = _al(eng._arena.data_ptr())
        end = eng._arena.data_ptr() + eng._arena.numel()
        if eng._ws is None:
            eng._ws = torch.empty(192 << 20, dtype=torch.uint8, device=dev)
        eng._ws_a, eng._ws_bytes = eng._ws.data_ptr(), eng._ws.numel()
        eng._stream = torch.cuda.current_stream().cuda_stream
        eng._fn = C.lib().osb_conv_fwd_tc
        eng._chain_on = False
        eng._flags = 1 if eng.use_pdl else 0
        need_bs = max(C.lib().osb_bn_stats_workspace_bytes(nl, eng._bs_cmax) for nl in n)
        if eng._bs_ws is None or eng._bs_ws.numel() < need_bs:
            eng._bs_ws = None
            eng._bs_ws = torch.empty(max(need_bs, 256), dtype=torch.uint8, device=dev)
        eng._bs_ws_a, eng._bs_ws_bytes = eng._bs_ws.data_ptr(), eng._bs_ws.numel()
        lib = C.lib()
        stats_fn, apply_fn = lib.osb_bn_batch_stats_save, lib.osb_bn_apply_split_out

        def alloc(rows_, c):
            a = eng._cursor
            eng._cursor += _al(rows_ * 4 * c)
            return a

        def norm(cv, z, rows_, y=None, res=0, res_cv=None):
            """statistics of z (saved mean / invstd, running buffers moved); y = relu(BN(z) + r) unless y is False"""
            bn = cv.bn
            w_a, b_a, rm_a, rv_a, nbt_a = cv.bs_args
            rc = stats_fn(z, rows_, cv.cout, w_a, b_a, bn.eps, -1.0 if bn.momentum is None else bn.momentum, rm_a, rv_a, nbt_a,
                          cv.bs_scale_a, cv.bs_shift_a, cv.bs_mean_a, cv.bs_invstd_a, eng._bs_ws_a, eng._bs_ws_bytes, eng._stream)
            if rc:
                C.check(rc, 'osb_bn_batch_stats_save')
            if y is False:
                return 0
            y = alloc(rows_, cv.cout)
            rc = apply_fn(z, y, rows_, cv.cout, cv.bs_scale_a, cv.bs_shift_a, res, res_cv.bs_scale_a if res_cv else 0,
                          res_cv.bs_shift_a if res_cv else 0, 1, eng._stream)
            if rc:
                C.check(rc, 'osb_bn_apply_split_out')
            return y

        tape = []

        def stage(blocks, srcs, lvl):
            x = srcs
            for (c1, c2, ds) in blocks:
                z1 = eng._conv(c1, x, nbr3[lvl][0], n[lvl], relu=0)
                y1 = norm(c1, z1, n[lvl])
                n1 = _Node(c1, z1, y1, n[lvl], x, 27, nbr3[lvl][0], nbr3[lvl][1])
                nd = None
                r, r_cv = x[0][0], None
                if ds is not None:
                    zd = eng._conv(ds, x, 0, n[lvl], relu=0)
                    norm(ds, zd, n[lvl], y=False)
                    nd = _Node(ds, zd, 0, n[lvl], x, 1, 0, 0)
                    r, r_cv = zd, ds
                z2 = eng._conv(c2, [(y1, c1.cout, n[lvl])], nbr3[lvl][0], n[lvl], relu=0)
                y2 = norm(c2, z2, n[lvl], res=r, res_cv=r_cv)
                n2 = _Node(c2, z2, y2, n[lvl], [(y1, c1.cout, n[lvl])], 27, nbr3[lvl][0], nbr3[lvl][1])
                tape.append(('block', (n1, nd, n2)))
                x = [(y2, c2.cout, n[lvl])]
            return x[0]

        cs0 = cm.sets[1].ensure_lookup()
        f32 = feats.detach().float().contiguous()
        x_int = torch.empty_like(f32)
        C.call('osb_gather_rows_f32', C.ptr(f32), C.ptr(cm.perm), n[0], f32.shape[1], C.ptr(x_int), C.stream_ptr())
        z0 = alloc(n[0], st.cout)
        if cs0.grid is not None:
            C.call('osb_conv_stem_fused_grid', C.ptr(x_int), st.cin, C.ptr(cs0.coords), n[0], C.ptr(cs0.grid), *cs0.grid_args,
                   st.ks, 1, C.ptr(st.w3), st.cout, 0, 0, 0, z0, None, eng._stream)
        else:
            C.call('osb_conv_stem_fused', C.ptr(x_int), st.cin, C.ptr(cs0.coords), n[0], C.ptr(cs0.slots), cs0.cap, st.ks, 1,
                   C.ptr(st.w3), st.cout, 0, 0, 0, z0, None, eng._stream)
        y0 = norm(st, z0, n[0])
        tape.append(('layer', _Node(st, z0, y0, n[0], [], st.K, k5.nbr.data_ptr(), 0, stem=True)))
        skips = [(y0, st.cout, n[0])]
        cur = skips[0]
        for l, (dconv, blocks) in enumerate(eng.enc):
            z = eng._conv(dconv, [cur], dn[l][0], n[l + 1], relu=0)
            y = norm(dconv, z, n[l + 1])
            nd = _Node(dconv, z, y, n[l + 1], [cur], 8, dn[l][0], dn[l][1])
            tape.append(('layer', nd))
            cur = stage(blocks, [(y, dconv.cout, n[l + 1])], l + 1)
            skips.append(cur)
        for j, (uconv, blocks) in enumerate(eng.dec):
            l = 3 - j
            z = alloc(n[l], uconv.cout)
            if eng.layer_log is not None:
                eng.layer_log.append((n[l + 1], 1, cur[1], uconv.K * uconv.cout, 'dense-up'))
            if eng.dense_up:
                rc = lib.osb_convtr_fwd_tc(cur[0], cur[1], n[l + 1], dn[l][0], uconv.K, uconv.wpack_a, uconv.cout, 0, 0, 0, z, 0,
                                           eng._flags, eng._stream)
                if rc:
                    C.check(rc, 'osb_convtr_fwd_tc')
            else:
                eng._cursor -= _al(n[l] * 4 * uconv.cout)
                z = eng._conv(uconv, [cur], dn[l][1], n[l], relu=0)
            y = norm(uconv, z, n[l])
            # transposed conv: forward map = the transposed down map (n_out fine rows), dgrad over the down map itself
            tape.append(('layer', _Node(uconv, z, y, n[l], [cur], uconv.K, dn[l][1], dn[l][0])))
            cur = stage(blocks, [(y, uconv.cout, n[l]), skips[l]], l)
        if eng._cursor > end:
            raise RuntimeError("forward_train: activation arena overflow (plan_train_bytes out of date)")
        fin = eng.final
        if cos is not None:
            out = _cos_forward(eng, cur, n[0], sel, cos, tape)
        elif l1 is not None:
            out = _l1_forward(eng, cur, n[0], sel, l1, tape)
        elif ce is None:
            out = torch.empty((m, fin.cout), dtype=torch.float32, device=dev)
            rc = eng._fn(cur[0], cur[1], n[0], 0, 0, 0, sel.data_ptr(), m, 1, fin.wpack_a, fin.cout, 0, 0, 0, 0, 0, out.data_ptr(),
                         0, eng._ws_a, eng._ws_bytes, eng._flags, eng._stream)
            if rc:
                C.check(rc, 'osb_conv_fwd_tc')
            tape.append(('head', _Node(fin, 0, 0, n[0], [cur], 1, sel.data_ptr(), sel_t.data_ptr())))
        else:
            out = _ce_forward(eng, cm, cur, n[0], ce, tape)
        if eng.layer_log is not None:
            eng.layer_log.append((m, 1, cur[1], fin.cout, 'head'))
    torch.autograd.graph.increment_version(eng._bs_tensors)
    gr = _Graph()
    gr.out, gr.tape, gr.gen, gr.n, gr.m = out, tape, eng._gen, n, m
    # everything the recorded addresses point into stays alive until the backward
    gr.keep = (cm, sel, sel_t, k5, eng._arena, eng._bs_buf, list(eng._bwd_convs), eng.stem)
    gr.x_pad = torch.nn.functional.pad(x_int, (0, 32 - x_int.shape[1]))      # stem wgrad operand (see _run_backward)
    return gr


def plan_buckets(tape, params):
    """[(lo, hi, t)]: all-reduce buckets over params[lo:hi], in the order the backward completes them (from the end of the
    parameter list, DistributedDataParallel's size caps), each issued after item t of the reversed tape, the item that writes
    the last of its slots."""
    index = {id(p): i for i, p in enumerate(params)}
    last = [None] * len(params)
    for t, (kind, item) in enumerate(reversed(tape)):
        nodes = item if kind == 'block' else (item[0] if kind in ('ce_head', 'cos_head', 'l1_head') else item,)
        for nd in nodes:
            if nd is not None:
                bn = nd.cv.bn
                for p in (nd.cv.mod.kernel,) + ((bn.weight, bn.bias) if bn is not None else ()):
                    last[index[id(p)]] = t
    if None in last:
        raise RuntimeError(f"forward_train backward: no tape item writes the gradient of parameter {last.index(None)}")
    out, hi, size, cap = [], len(params), 0, _FIRST_BUCKET_BYTES
    for i in range(len(params) - 1, -1, -1):
        size += 4 * params[i].numel()
        if size >= cap or i == 0:
            out.append((i, hi, max(last[i:hi])))
            hi, size, cap = i, 0, _BUCKET_BYTES
    return out


def _run_backward(eng, gr, g, params):
    if gr.gen != eng._gen:
        raise RuntimeError("FusedMinkUNet: the activations saved by forward_train were overwritten by a later forward / "
                           "forward_train on the same engine; run backward before the next forward")
    dev = eng.device
    lib = C.lib()
    stream = torch.cuda.current_stream().cuda_stream
    g = g.detach().float().contiguous()
    # one flat buffer for all parameter gradients; every slot is written by exactly one launch below
    index = {id(p): i for i, p in enumerate(params)}
    flat = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
    views, offs = [], [0]
    for p in params:
        views.append(flat[offs[-1]:offs[-1] + p.numel()].view(p.shape))
        offs.append(offs[-1] + p.numel())
    written = [False] * len(params)
    pg = eng.process_group
    buckets = plan_buckets(gr.tape, params) if pg is not None else []
    world = dist.get_world_size(group=pg) if pg is not None else 1
    works = []

    def issue(t):
        """all-reduce every bucket whose last slot tape item t wrote: g / world on every rank, summed"""
        while len(works) < len(buckets) and buckets[len(works)][2] == t:
            lo, hi, _ = buckets[len(works)]
            if not all(written[lo:hi]):
                raise RuntimeError(f"forward_train backward: the gradient bucket of parameters {lo}..{hi - 1} is due after "
                                   f"tape item {t} with {hi - lo - sum(written[lo:hi])} slots still unwritten")
            b = flat[offs[lo]:offs[hi]]
            b.div_(world)
            works.append(dist.all_reduce(b, group=pg, async_op=True))

    def slot(p):
        i = index[id(p)]
        if written[i]:
            raise RuntimeError("forward_train backward: a parameter gradient written twice")
        written[i] = True
        return views[i]

    # grow-only chunks of gradient rows, reused by every backward (stream-ordered)
    pool = eng._garena
    state = {'chunk': 0, 'cur': 0}
    if pool:
        state['cur'] = _al(pool[0].data_ptr())

    def galloc(nbytes):
        nbytes = _al(nbytes)
        while True:
            i = state['chunk']
            if i == len(pool):
                pool.append(torch.empty(max(_GCHUNK, nbytes + 256), dtype=torch.uint8, device=dev))
                state['cur'] = _al(pool[i].data_ptr())
            t = pool[i]
            if state['cur'] + nbytes <= t.data_ptr() + t.numel():
                a = state['cur']
                state['cur'] += nbytes
                return a
            state['chunk'] = i + 1
            if state['chunk'] < len(pool):
                state['cur'] = _al(pool[state['chunk']].data_ptr())

    sums = torch.empty(2 * eng._bs_cmax, dtype=torch.float32, device=dev)
    sums_a = sums.data_ptr()
    wg_ws = [None]

    def wg_workspace(nbytes):
        if wg_ws[0] is None or wg_ws[0].numel() < nbytes:
            wg_ws[0] = None
            wg_ws[0] = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
        return wg_ws[0].data_ptr(), wg_ws[0].numel()

    grads = {}

    def bn_bwd(nd, gin, y_mask, gp=0, gp_acc=0):
        cv, bn = nd.cv, nd.cv.bn
        rc = lib.osb_bn_backward_reduce(y_mask, gin, nd.z, nd.n, cv.cout, cv.bs_mean_a, cv.bs_invstd_a, sums_a,
                                        slot(bn.weight).data_ptr(), slot(bn.bias).data_ptr(), 0, eng._bs_ws_a, eng._bs_ws_bytes,
                                        stream)
        if rc:
            C.check(rc, 'osb_bn_backward_reduce')
        dz = galloc(nd.n * 4 * cv.cout)
        rc = lib.osb_bn_backward_apply(y_mask, gin, nd.z, nd.n, cv.cout, cv.bs_mean_a, cv.bs_invstd_a, cv.bs_args[0], sums_a, dz,
                                       gp, gp_acc, stream)
        if rc:
            C.check(rc, 'osb_bn_backward_apply')
        return dz

    def conv_bwd(nd, dz, n_out):
        """wgrad into the kernel's gradient slot, dgrad contributions to every source"""
        cv = nd.cv
        widths = [c for (_, c, _) in nd.srcs]
        gk = slot(cv.mod.kernel)
        K = nd.K
        gk3 = gk.view(K, cv.cin, cv.cout)
        for (lo, hi, _), (src, c, n_in) in zip(_packs_for(cv, widths), nd.srcs):
            gw = gk3 if len(widths) == 1 else torch.empty((K, c, cv.cout), dtype=torch.float32, device=dev)
            ws_a, ws_b = wg_workspace(lib.osb_conv_wgrad_tc_workspace_bytes(n_out, K, c, cv.cout))
            rc = lib.osb_conv_wgrad_tc(src, c, n_in, nd.nbr_f, n_out, K, dz, cv.cout, gw.data_ptr(), ws_a, ws_b, stream)
            if rc:
                C.check(rc, 'osb_conv_wgrad_tc')
            if len(widths) > 1:
                gk3[:, lo:hi].copy_(gw)
        for (lo, hi, pk), (src, c, n_in) in zip(_packs_for(cv, widths), nd.srcs):
            res = grads.get(src, 0)
            out = galloc(n_in * 4 * c)
            rc = lib.osb_conv_fwd_tc(dz, cv.cout, n_out, 0, 0, 0, nd.nbr_b, n_in, K, pk.data_ptr(), c, 0, 0, res, 0, out, 0, 0,
                                     eng._ws_a, eng._ws_bytes, 0, stream)
            if rc:
                C.check(rc, 'osb_conv_fwd_tc')
            grads[src] = out

    with torch.cuda.device(dev):
        for t, (kind, item) in enumerate(reversed(gr.tape)):
            if kind == 'head':
                nd = item
                cv = nd.cv
                gs = galloc(gr.m * 4 * cv.cout)
                C.call('osb_f32_to_split', C.ptr(g), gr.m, cv.cout, gs, C.stream_ptr())
                (src, c, n0), = nd.srcs
                gw = slot(cv.mod.kernel)
                ws_a, ws_b = wg_workspace(lib.osb_conv_wgrad_tc_workspace_bytes(gr.m, 1, c, cv.cout))
                rc = lib.osb_conv_wgrad_tc(src, c, n0, nd.nbr_f, gr.m, 1, gs, cv.cout, gw.data_ptr(), ws_a, ws_b, stream)
                if rc:
                    C.check(rc, 'osb_conv_wgrad_tc')
                (_, _, pk), = _packs_for(cv, [c])
                out = galloc(n0 * 4 * c)
                rc = lib.osb_conv_fwd_tc(gs, cv.cout, gr.m, 0, 0, 0, nd.nbr_b, n0, 1, pk.data_ptr(), c, 0, 0, 0, 0, out, 0, 0,
                                         eng._ws_a, eng._ws_bytes, 0, stream)
                if rc:
                    C.check(rc, 'osb_conv_fwd_tc')
                grads[src] = out
            elif kind == 'ce_head':
                _ce_backward(eng, item, g, slot, galloc, grads, stream)
            elif kind == 'cos_head':
                _cos_backward(eng, item, g, slot, galloc, grads, stream)
            elif kind == 'l1_head':
                _l1_backward(eng, item, g, slot, galloc, grads, stream)
            elif kind == 'block':
                n1, nd_, n2 = item
                g2 = grads[n2.y]
                x = n1.srcs
                gp, gp_acc = 0, 0
                if nd_ is None:                                  # identity shortcut: the block input receives g'
                    src = x[0][0]
                    gp_acc = 1 if src in grads else 0
                    gp = grads[src] if gp_acc else galloc(n2.n * 4 * n2.cv.cout)
                    grads[src] = gp
                dz2 = bn_bwd(n2, g2, n2.y, gp, gp_acc)
                if nd_ is not None:                              # downsample: its BatchNorm sees g' through the same mask
                    dzd = bn_bwd(nd_, g2, n2.y)
                    conv_bwd(nd_, dzd, nd_.n)
                conv_bwd(n2, dz2, n2.n)
                dz1 = bn_bwd(n1, grads[n1.y], n1.y)
                conv_bwd(n1, dz1, n1.n)
            else:
                nd = item
                dz = bn_bwd(nd, grads[nd.y], nd.y)
                if nd.stem:
                    # the 3 input channels zero-padded to one 32-channel split line: the fixed-order tensor-core wgrad
                    # (osb_conv_wgrad_f32 adds with float atomics, so two identical steps would differ in the last bits)
                    cv = nd.cv
                    xs = galloc(nd.n * 4 * 32)
                    C.call('osb_f32_to_split', C.ptr(gr.x_pad), nd.n, 32, xs, C.stream_ptr())
                    gw = torch.empty((cv.K, 32, cv.cout), dtype=torch.float32, device=dev)
                    ws_a, ws_b = wg_workspace(lib.osb_conv_wgrad_tc_workspace_bytes(nd.n, cv.K, 32, cv.cout))
                    rc = lib.osb_conv_wgrad_tc(xs, 32, nd.n, nd.nbr_f, nd.n, cv.K, dz, cv.cout, gw.data_ptr(), ws_a, ws_b, stream)
                    if rc:
                        C.check(rc, 'osb_conv_wgrad_tc')
                    slot(cv.mod.kernel).copy_(gw[:, :cv.cin])
                else:
                    conv_bwd(nd, dz, nd.n)
            if buckets:
                issue(t)
        for w in works:
            w.wait()
    missing = [i for i, w in enumerate(written) if not w]
    if missing:
        raise RuntimeError(f"forward_train backward: {len(missing)} parameters without a gradient")
    gr.keep = None
    return views
