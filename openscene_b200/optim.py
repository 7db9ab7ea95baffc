"""Adam and SGD whose step runs on the device and leaves a bound training engine ready for its next forward.

``Adam`` and ``SGD`` are drop-in ``torch.optim.Optimizer`` subclasses for the two optimisers the reference's training drivers
use (run/distill.py: Adam with a poly learning rate written into ``param_groups``; run/train_mink.py: SGD with momentum 0.9 and
weight decay 1e-4).  ``step()`` updates every parameter that has a gradient in ONE launch (``osb_optim_adam`` /
``osb_optim_sgd``, csrc/optim.cu) with torch's foreach arithmetic, and keeps ``state`` in torch's layout, so checkpoints move
between these classes and ``torch.optim.Adam`` / ``SGD`` in either direction.

``opt.bind(engine)`` attaches a ``FusedMinkUNet(model, batch_stats=True)`` whose parameters the optimiser holds.  After the
update, ``step()`` re-packs the engine's split-bf16 operands in place (one ``osb_conv_repack`` over
``engine.repack_jobs()``) and marks the engine current, so its next forward does not rebuild itself through ``refresh()``.
Every written tensor's version is bumped, so other consumers of the same parameters (an eval engine, ``fast_eval``, the
module path's pack cache, autograd's in-place check) see the write.  Nothing synchronises with the host: the tables go up as
one pinned host-to-device copy each, stream-ordered on the current stream."""
import numpy as np
import torch
from torch.optim.optimizer import _get_scalar_dtype

from . import _cabi as C

OPTIM_CHUNK = 16384                      # elements of one tensor per block of the update kernels
PACK_CHUNK = 8192                        # packed elements of one job per block of osb_conv_repack

_ADAM = np.dtype([('param', '<u8'), ('grad', '<u8'), ('exp_avg', '<u8'), ('exp_avg_sq', '<u8'), ('numel', '<i8'),
                  ('chunk_begin', '<i8'), ('step_size', '<f4'), ('bc2_sqrt', '<f4'), ('lerp_w', '<f4'), ('beta2', '<f4'),
                  ('one_minus_beta2', '<f4'), ('eps', '<f4')])
_SGD = np.dtype([('param', '<u8'), ('grad', '<u8'), ('momentum_buffer', '<u8'), ('numel', '<i8'), ('chunk_begin', '<i8'),
                 ('neg_lr', '<f4'), ('weight_decay', '<f4'), ('momentum', '<f4'), ('first', '<i4')])
_JOB = np.dtype([('w', '<u8'), ('wpack', '<u8'), ('sk', '<i8'), ('sn', '<i8'), ('sc', '<i8'), ('chunk_begin', '<i8'),
                 ('K', '<i4'), ('cin', '<i4'), ('cout', '<i4'), ('cout_pad', '<i4')])
_LAYOUT_CHECKED = []


def _check_layouts():
    """the numpy records above against include/osb200.h's structs (once per process)"""
    if not _LAYOUT_CHECKED:
        for kind, dt in enumerate((_ADAM, _SGD, _JOB)):
            if C.lib().osb_optim_entry_bytes(kind) != dt.itemsize:
                raise RuntimeError(f"openscene_b200.optim: table entry {kind} is {dt.itemsize} bytes here, "
                                   f"{C.lib().osb_optim_entry_bytes(kind)} in libosb200 (header / binding mismatch)")
        _LAYOUT_CHECKED.append(True)


def _chunks(numel, chunk):
    """chunk_begin column and the total"""
    n = -(-np.asarray(numel, dtype=np.int64) // chunk)
    begin = np.zeros_like(n)
    np.cumsum(n[:-1], out=begin[1:])
    return begin, int(n.sum())


def _upload(table, device):
    """host records -> device table: one pinned host-to-device copy on the current stream (the caching host allocator keeps
    the pinned block until the copy has run)"""
    return torch.from_numpy(table.view(np.uint8)).pin_memory().to(device, non_blocking=True)


def repack_table(jobs):
    """engine.repack_jobs() -> (records, n_chunks) of osb_conv_repack"""
    t = np.zeros(len(jobs), dtype=_JOB)
    for i, (w, pk, (sk, sn, sc), K, cin, cout, pad) in enumerate(jobs):
        if pk.numel() != 4 * K * pad * cin:
            raise RuntimeError(f"repack job {i}: a pack of {pk.numel()} bytes for [{K}, {pad}, {cin}] rows")
        t[i] = (w.data_ptr(), pk.data_ptr(), sk, sn, sc, 0, K, cin, cout, pad)
    t['chunk_begin'], total = _chunks(t['K'].astype(np.int64) * t['cout_pad'] * t['cin'], PACK_CHUNK)
    return t, total


class _DeviceOptimizer(torch.optim.Optimizer):
    """What Adam and SGD share: refusals, engine binding, the pointer table and the launch."""
    _REFUSE = ()                          # (group key, value torch uses when the option is off)

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._engines = []
        self._engine_tables = {}          # id(engine) -> (jobs key, device table, n_jobs, n_chunks)
        self._addr = self._table = self._total = None      # the last update table, its addresses and chunk count

    def bind(self, engine):
        """Re-pack ``engine``'s tensor-core operands in place after every step (a ``FusedMinkUNet(model, batch_stats=True)``
        whose parameters are all in this optimiser).  An eval engine folds BatchNorm into its packs and re-folds by itself."""
        if not getattr(engine, 'batch_stats', False):
            raise ValueError("bind: the engine must be a FusedMinkUNet(model, batch_stats=True); an eval engine re-folds "
                             "BatchNorm from the running statistics by itself (refresh())")
        mine = {id(p) for g in self.param_groups for p in g['params']}
        missing = [n for n, p in engine._net.named_parameters() if id(p) not in mine]
        if missing:
            raise ValueError(f"bind: {len(missing)} engine parameters are not in this optimiser (first: {missing[0]})")
        if all(e is not engine for e in self._engines):
            self._engines.append(engine)
        return engine

    def _refuse_group(self, group):
        for key, off in self._REFUSE:
            if bool(group.get(key, off)) != bool(off):
                raise NotImplementedError(f"{type(self).__name__}: {key}={group[key]!r} is not implemented on the device "
                                          f"(the reference's training drivers never use it); use torch.optim")

    def _collect(self):
        """[(group, [params with a gradient])] after every refusal, before any work"""
        out, dev = [], None
        for group in self.param_groups:
            self._refuse_group(group)
            ps = []
            for p in group['params']:
                if p.grad is None:
                    continue
                g = p.grad
                if p.dtype != torch.float32 or not p.is_cuda or not p.is_contiguous():
                    raise NotImplementedError(f"{type(self).__name__}: parameters must be contiguous fp32 CUDA tensors "
                                              f"(got {p.dtype} on {p.device}, contiguous={p.is_contiguous()})")
                if g.is_sparse:
                    raise NotImplementedError(f"{type(self).__name__}: sparse gradients are not supported")
                if g.dtype != torch.float32 or g.device != p.device or not g.is_contiguous() or g.shape != p.shape:
                    raise NotImplementedError(f"{type(self).__name__}: gradients must be contiguous fp32 tensors shaped and "
                                              f"placed like their parameters")
                if dev is None:
                    dev = p.device
                elif p.device != dev:
                    raise NotImplementedError(f"{type(self).__name__}: parameters on several devices ({dev}, {p.device})")
                ps.append(p)
            out.append((group, ps))
        return out, dev

    def _engine_table(self, eng, dev):
        jobs = eng.repack_jobs()
        key = tuple((w.data_ptr(), pk.data_ptr(), s, K, cin, cout, pad) for (w, pk, s, K, cin, cout, pad) in jobs)
        ent = self._engine_tables.get(id(eng))
        if ent is None or ent[0] != key:
            t, total = repack_table(jobs)
            ent = self._engine_tables[id(eng)] = (key, _upload(t, dev), len(jobs), total)
        return ent

    def _records(self, dtype, addr, cols):
        """The update table: ``addr`` rows (pointers, numel) fill the leading fields, ``cols`` rows the per-tensor scalars.
        The pointer part is rebuilt only when an address changed since the last step; empty tensors are left out."""
        keep = [i for i, a in enumerate(addr) if a[-1] > 0]
        addr = [addr[i] for i in keep]
        if addr != self._addr:
            t = np.zeros(len(addr), dtype=dtype)
            for name, col in zip(dtype.names, zip(*addr)):
                t[name] = col
            t['chunk_begin'], self._total = _chunks(t['numel'], OPTIM_CHUNK)
            self._addr, self._table = addr, t
        t = self._table
        scalar_names = dtype.names[len(addr[0]) + 1:] if addr else ()
        for name, col in zip(scalar_names, zip(*[cols[i] for i in keep])):
            t[name] = col
        return t

    def _launch(self, name, table, dev, written):
        """the update over all groups, the version bumps, then one re-pack per bound engine"""
        _check_layouts()
        stale = [e for e in self._engines if e._sig != e._signature()]     # changed behind our back: left to refresh()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream().cuda_stream
            if len(table):
                tab = _upload(table, dev)
                C.check(getattr(C.lib(), name)(tab.data_ptr(), len(table), OPTIM_CHUNK, self._total, stream), name)
        torch.autograd.graph.increment_version(written)
        self.repack_bound([e for e in self._engines if not any(e is s for s in stale)])

    def repack_bound(self, engines=None):
        """Re-pack the bound engines (default: all) in place from their module's current weights and mark them current;
        ``step()`` does this after its update.  One ``osb_conv_repack`` launch per engine, on the current stream."""
        engines = self._engines if engines is None else engines
        for eng in engines:
            with torch.cuda.device(eng.device):
                _, jt, nj, nc = self._engine_table(eng, eng.device)
                jt.record_stream(torch.cuda.current_stream())
                C.check(C.lib().osb_conv_repack(jt.data_ptr(), nj, PACK_CHUNK, nc, torch.cuda.current_stream().cuda_stream),
                        'osb_conv_repack')
            eng._sig = eng._signature()


class Adam(_DeviceOptimizer):
    """``torch.optim.Adam(params, lr, betas, eps)`` (weight_decay 0, no amsgrad / maximize) with the update on the device."""
    _REFUSE = (('amsgrad', False), ('maximize', False), ('weight_decay', 0), ('capturable', False),
               ('differentiable', False), ('fused', None), ('decoupled_weight_decay', False))

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize,
                        foreach=foreach, capturable=capturable, differentiable=differentiable, fused=fused,
                        decoupled_weight_decay=decoupled_weight_decay)
        for key, off in self._REFUSE:                     # refuse at construction as well as at every step
            if bool(defaults[key]) != bool(off):
                raise NotImplementedError(f"Adam: {key}={defaults[key]!r} is not implemented on the device (the reference's "
                                          f"training drivers never use it); use torch.optim.Adam")
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        groups, dev = self._collect()
        rows = [(group, p, self.state[p]) for group, ps in groups for p in ps]
        for _, p, st in rows:
            for k in ('exp_avg', 'exp_avg_sq'):
                t = st.get(k)
                if t is not None and (t.dtype != torch.float32 or t.device != p.device or not t.is_contiguous()
                                      or t.shape != p.shape):
                    raise NotImplementedError(f"Adam: state {k} must be a contiguous fp32 tensor like its parameter")
        for _, p, st in rows:
            if len(st) == 0:                              # torch.optim.Adam._init_group
                st['step'] = torch.tensor(0.0, dtype=_get_scalar_dtype())
                st['exp_avg'] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if not rows:
            return loss
        torch._foreach_add_([st['step'] for _, _, st in rows], torch.tensor(1.0, device='cpu'), alpha=1.0)   # torch's CPU counters
        scal, cols = {}, []
        for group, p, st in rows:
            lr, (beta1, beta2), eps = group['lr'], group['betas'], group['eps']
            key = (lr, beta1, beta2, eps, st['step'].item())
            s = scal.get(key)
            if s is None:
                # _multi_tensor_adam with capturable=False: Python doubles, each rounded to fp32 once in the table
                step = key[-1]
                bc1 = 1 - beta1 ** step
                bc2 = 1 - beta2 ** step
                s = scal[key] = ((lr / bc1) * -1, bc2 ** 0.5, 1 - beta1, beta2, 1 - beta2, eps)
            cols.append(s)
        table = self._records(_ADAM, [(p.data_ptr(), p.grad.data_ptr(), st['exp_avg'].data_ptr(), st['exp_avg_sq'].data_ptr(),
                                       p.numel()) for _, p, st in rows], cols)
        written = [t for _, p, st in rows for t in (p, st['exp_avg'], st['exp_avg_sq'])]
        self._launch('osb_optim_adam', table, dev, written)
        return loss


class SGD(_DeviceOptimizer):
    """``torch.optim.SGD(params, lr, momentum, weight_decay)`` (no dampening / nesterov / maximize) with the update on the
    device."""
    _REFUSE = (('dampening', 0), ('nesterov', False), ('maximize', False), ('differentiable', False), ('fused', None))

    def __init__(self, params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False, *, maximize=False,
                 foreach=None, differentiable=False, fused=None):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                        maximize=maximize, foreach=foreach, differentiable=differentiable, fused=fused)
        for key, off in self._REFUSE:
            if bool(defaults[key]) != bool(off):
                raise NotImplementedError(f"SGD: {key}={defaults[key]!r} is not implemented on the device (the reference's "
                                          f"training drivers never use it); use torch.optim.SGD")
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        groups, dev = self._collect()
        rows = []
        for group, ps in groups:
            for p in ps:
                buf = self.state[p].get('momentum_buffer') if group['momentum'] != 0 else None
                if buf is not None and (buf.dtype != torch.float32 or buf.device != p.device or not buf.is_contiguous()
                                        or buf.shape != p.shape):
                    raise NotImplementedError("SGD: momentum_buffer must be a contiguous fp32 tensor like its parameter")
                rows.append((group, p, buf))
        if not rows:
            return loss
        addr, cols, written = [], [], []
        for group, p, buf in rows:
            first = 0
            if group['momentum'] != 0:
                if buf is None:                           # torch: a clone of the first (decayed) gradient
                    buf = self.state[p]['momentum_buffer'] = torch.empty_like(p)
                    first = 1
                written.append(buf)
            addr.append((p.data_ptr(), p.grad.data_ptr(), buf.data_ptr() if buf is not None else 0, p.numel()))
            cols.append((-group['lr'], group['weight_decay'], group['momentum'], first))
            written.append(p)
        self._launch('osb_optim_sgd', self._records(_SGD, addr, cols), dev, written)
        return loss
