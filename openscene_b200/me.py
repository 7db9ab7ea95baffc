"""The ``MinkowskiEngine`` surface OpenScene uses, re-implemented over ``libosb200`` (sm_90a).

Importable as ``MinkowskiEngine`` (the top-level ``MinkowskiEngine/`` package re-exports this
module) so that the reference's ``models/mink_unet.py``, ``models/resnet_base.py``,
``run/evaluate.py`` and ``run/distill.py`` work unchanged, and so that existing checkpoints load
with ``strict=True``: parameter / buffer names and shapes are the ones listed in SURVEY.md 8a
(``kernel`` of shape [K^3, Cin, Cout] or [Cin, Cout] for 1x1x1; ``bn.*`` under MinkowskiBatchNorm).

Reference call sites: models/mink_unet.py:25-26,47-114; models/resnet_base.py:27-28,73-118;
run/evaluate.py:18,284; run/distill.py:18,316.
"""
import math

import torch
import torch.nn as nn

from . import _cabi as C
from .coords import CoordinateManager

__version__ = '0.5.4+osb200'


class CoordinateMapKey:
    def __init__(self, tensor_stride, string_id=''):
        self.ts = int(tensor_stride)
        self.string_id = string_id

    def get_tensor_stride(self):
        return [self.ts] * 3

    def __eq__(self, o):
        return isinstance(o, CoordinateMapKey) and o.ts == self.ts and o.string_id == self.string_id

    def __hash__(self):
        return hash((self.ts, self.string_id))

    def __repr__(self):
        return f"CoordinateMapKey(tensor_stride={[self.ts] * 3})"


class SparseTensor:
    """``ME.SparseTensor(features, coordinates)`` -- features first (run/evaluate.py:284).

    Rows of ``.F`` / ``.C`` at tensor stride 1 are in the caller's order (the drivers index the
    network output with ``inds_reverse`` / ``mask``: run/evaluate.py:290, run/distill.py:322).
    Internally features live in Morton row order (``_F``)."""

    def __init__(self, features, coordinates=None, tensor_stride=1, coordinate_map_key=None,
                 coordinate_manager=None, quantization_mode=None, device=None, **kwargs):
        if device is not None:
            features = features.to(device)
        C.require_cuda(features, 'SparseTensor features')
        self._cm = self._raw_coords = self._Fi = None
        if coordinate_manager is None:
            if coordinates is None:
                raise ValueError("SparseTensor needs coordinates or a coordinate_manager")
            ts = tensor_stride if isinstance(tensor_stride, int) else int(tensor_stride[0])
            if ts != 1:
                raise NotImplementedError("SparseTensor from raw coordinates supports tensor_stride=1 only")
            if coordinates.dim() != 2 or coordinates.shape[1] != 4:
                raise ValueError("coordinates must be [N,4] (batch, x, y, z)")
            if features.shape[0] != coordinates.shape[0]:
                raise ValueError(f"features have {features.shape[0]} rows, coordinates have {coordinates.shape[0]}")
            # The coordinate manager (sort, lookup structures) and the internal-order copy of the features are built on
            # first use: the fused eval path (fast_eval.py) builds the whole encoder pyramid in one native call instead.
            self._raw_coords = coordinates.to(features.device)
            self.coordinate_map_key = CoordinateMapKey(1)
            self._F_ext = features
            self._split = None
            if not torch.is_grad_enabled():
                from . import fast_eval
                fast_eval.watch(self)
            return
        if coordinate_map_key is None:
            ts = tensor_stride if isinstance(tensor_stride, int) else int(tensor_stride[0])
            coordinate_map_key = CoordinateMapKey(ts)
        self._cm = coordinate_manager
        self.coordinate_map_key = coordinate_map_key
        n = coordinate_manager.sets[coordinate_map_key.ts].n
        if features.shape[0] != n:
            raise ValueError(f"features have {features.shape[0]} rows, coordinate set has {n}")
        self._Fi = _to_internal(features, coordinate_manager, coordinate_map_key.ts)
        self._F_ext = features if coordinate_map_key.ts == 1 else None
        self._split = None

    # -- lazily built state ------------------------------------------------------------------
    @property
    def coordinate_manager(self):
        if self._cm is None:
            self._cm = CoordinateManager(self._raw_coords)
        return self._cm

    @coordinate_manager.setter
    def coordinate_manager(self, cm):
        self._cm = cm

    @property
    def _F(self):
        """features in internal (Morton) row order"""
        if self._Fi is None:
            self._Fi = _to_internal(self._F_ext, self.coordinate_manager, self.coordinate_map_key.ts)
        return self._Fi

    @_F.setter
    def _F(self, v):
        self._Fi = v

    def _is_fresh_input(self):
        """an input tensor straight from ``SparseTensor(features, coordinates)`` that nothing has consumed or modified"""
        return self._raw_coords is not None and self._Fi is None and self._F_ext is not None

    # -- internal constructors ---------------------------------------------------------------
    @classmethod
    def _wrap(cls, F_int, cm, ts):
        t = cls.__new__(cls)
        t._cm, t._raw_coords, t.coordinate_map_key = cm, None, CoordinateMapKey(ts)
        t._Fi, t._F_ext, t._split = F_int, None, None
        return t

    # -- public surface ------------------------------------------------------------------------
    @property
    def _ts(self):
        return self.coordinate_map_key.ts

    @property
    def F(self):
        if self._ts != 1:
            return self._F
        if self._F_ext is None:
            self._F_ext = _to_external(self._F, self.coordinate_manager)
        return self._F_ext

    @property
    def feats(self):
        return self.F

    @property
    def C(self):
        return self.coordinate_manager.coords_external(self._ts)

    @property
    def coordinates(self):
        return self.C

    @property
    def tensor_stride(self):
        return [self._ts] * 3

    @property
    def D(self):
        return 3

    def _any_F(self):
        return self._Fi if self._Fi is not None else self._F_ext

    @property
    def device(self):
        return self._any_F().device

    @property
    def dtype(self):
        return self._any_F().dtype

    @property
    def shape(self):
        return self._any_F().shape

    def size(self, *a):
        return self._any_F().size(*a)

    def __len__(self):
        return self._any_F().shape[0]

    def _same_set(self, o):
        if o.coordinate_manager is not self.coordinate_manager or o._ts != self._ts:
            raise ValueError("SparseTensors live on different coordinate sets")

    def __add__(self, o):
        self._same_set(o)
        return SparseTensor._wrap(self._F + o._F, self.coordinate_manager, self._ts)

    def __iadd__(self, o):
        self._same_set(o)
        self._F = self._F + o._F
        self._F_ext = None
        self._split = None
        return self

    def __sub__(self, o):
        self._same_set(o)
        return SparseTensor._wrap(self._F - o._F, self.coordinate_manager, self._ts)

    def __mul__(self, o):
        self._same_set(o)
        return SparseTensor._wrap(self._F * o._F, self.coordinate_manager, self._ts)

    def __repr__(self):
        return f"SparseTensor(N={self.shape[0]}, C={self.shape[1]}, tensor_stride={self.tensor_stride})"


def _require_f32(t, what):
    """The CUDA-core entry points read fp32 rows: any other dtype would be reinterpreted (fp64) or read and written out of
    bounds (fp16), so it is refused before anything launches."""
    if t.dtype != torch.float32:
        raise TypeError(f"openscene_b200: {what} must be float32, got {t.dtype}")


class _RowGather(torch.autograd.Function):
    """out[r] = x[idx[r]] with idx a permutation (its inverse ``inv`` drives the backward)."""

    @staticmethod
    def forward(ctx, x, idx, inv):
        _require_f32(x, 'row gather input')
        ctx.save_for_backward(idx, inv)
        x = x.contiguous()
        out = torch.empty_like(x)
        C.call('osb_gather_rows_f32', C.ptr(x), C.ptr(idx), x.shape[0], x.shape[1], C.ptr(out), C.stream_ptr())
        return out

    @staticmethod
    def backward(ctx, g):
        idx, inv = ctx.saved_tensors
        return _RowGather.apply(g, inv, idx), None, None


def _to_internal(F_ext, cm, ts):
    if ts != 1:
        return F_ext
    F32 = F_ext if F_ext.dtype == torch.float32 else F_ext.float()
    return _RowGather.apply(F32, cm.perm, cm.inv_perm)


def _to_external(F_int, cm):
    return _RowGather.apply(F_int, cm.inv_perm, cm.perm)


def cat(*tensors):
    """``ME.cat(a, b)``: column concatenation on one coordinate set (mink_unet.py:147,155,163,171)."""
    if len(tensors) == 1 and isinstance(tensors[0], (list, tuple)):
        tensors = tuple(tensors[0])
    t0 = tensors[0]
    for t in tensors[1:]:
        t0._same_set(t)
    return SparseTensor._wrap(torch.cat([t._F for t in tensors], dim=1), t0.coordinate_manager, t0._ts)


# ------------------------------------------------------------------------------------------------
# sparse convolution: out[o,:] = sum_k in[nbr[k][o],:] @ W[k]
# ------------------------------------------------------------------------------------------------
def _conv_raw(x, kmap, w3, n_out, transpose_w=False):
    """x fp32 [n_in, cin]; w3 fp32 [K, cin, cout] ([K, cout, cin] when transpose_w)."""
    _require_f32(x, 'convolution input')
    _require_f32(w3, 'convolution kernel')
    x = x.contiguous()
    w3 = w3.contiguous()
    K = w3.shape[0]
    cin, cout = (w3.shape[2], w3.shape[1]) if transpose_w else (w3.shape[1], w3.shape[2])
    assert x.shape[1] == cin, f"conv expects {cin} input channels, got {x.shape[1]}"
    out = torch.empty((n_out, cout), dtype=torch.float32, device=x.device)
    nbr = kmap.nbr if kmap is not None else None
    C.call('osb_conv_fwd_f32', C.ptr(x), cin, C.ptr(nbr), n_out, K, C.ptr(w3), cin, cout, int(transpose_w),
           C.ptr(out), C.stream_ptr())
    return out


def _tc_ok(cin, cout, K):
    return cin % 32 == 0 and cout % 32 == 0 and K <= 32 and _module_tc_enabled()


def _conv_tc_split(xs, kmap, wpack, cin, cout, K, n_out):
    """split rows in, fp32 rows out through the tensor-core kernel (bf16x3 split operands)."""
    from . import tc
    nbr = kmap.nbr if kmap is not None else None
    return tc.conv_tc(xs, cin, None, 0, nbr, n_out, K, wpack, cout, out_split=False, out_f32=True)[1]


class SparseConvFunction(torch.autograd.Function):
    """Forward / dgrad / wgrad of the generalised sparse convolution on libosb200 kernels
    (replaces MinkowskiConvolutionFunction / ...TransposeFunction inside MinkowskiEngine; run/distill.py:321,333).
    With channel counts that are multiples of 32 all three run on tensor cores: forward and dgrad on the tensor-core
    convolution kernel (dgrad = the same kernel on the transposed map with W^T packed), wgrad on csrc/conv_wgrad_tc.cu.
    The input is saved in the split-bf16 layout the kernels read (the conversion is paid once, in forward); packed weights
    are memoised on the parameter's version counter.  Odd shapes use the exact-fp32 CUDA-core kernels."""

    @staticmethod
    def forward(ctx, x, w3, kmap, n_out):
        ctx.kmap, ctx.n_in = kmap, x.shape[0]
        K, cin, cout = w3.shape
        ctx.tc = bool(_tc_ok(cin, cout, K) and x.dtype == torch.float32)
        with torch.cuda.device(x.device):
            if ctx.tc:
                from . import tc
                xs = tc.to_split(x.contiguous())
                ctx.save_for_backward(xs, w3)
                return _conv_tc_split(xs, kmap, tc.packed_weights_cached(w3), cin, cout, K, n_out)
            ctx.save_for_backward(x, w3)
            return _conv_raw(x, kmap, w3, n_out)

    @staticmethod
    def backward(ctx, gout):
        x, w3 = ctx.saved_tensors
        kmap = ctx.kmap
        gout = gout.contiguous()
        gx = gw = None
        K, cin, cout = w3.shape
        with torch.cuda.device(gout.device):
            if ctx.tc and gout.dtype == torch.float32:
                from . import tc
                gs = tc.to_split(gout)                                    # shared by dgrad and wgrad
                if ctx.needs_input_grad[0]:
                    kt = kmap.transposed() if kmap is not None else None
                    gx = _conv_tc_split(gs, kt, tc.packed_weights_cached(w3, transpose_w=True), cout, cin, K, ctx.n_in)
                if ctx.needs_input_grad[1]:
                    nbr = kmap.nbr if kmap is not None else None
                    gw = tc.conv_wgrad_tc(x, cin, ctx.n_in, nbr, gout.shape[0], K, gs, cout)
                return gx, gw, None, None
            if ctx.tc:                                                    # saved input is in the split layout
                from . import tc
                x = tc.from_split(x, cin)
            if ctx.needs_input_grad[0]:
                kt = kmap.transposed() if kmap is not None else None
                gx = _conv_raw(gout, kt, w3, ctx.n_in, transpose_w=True)
            if ctx.needs_input_grad[1]:
                _require_f32(x, 'convolution input')
                _require_f32(gout, 'convolution output gradient')
                _require_f32(w3, 'convolution kernel')
                gw = torch.empty_like(w3)
                nbr = kmap.nbr if kmap is not None else None
                C.call('osb_conv_wgrad_f32', C.ptr(x.contiguous()), C.ptr(nbr), gout.shape[0], K, C.ptr(gout),
                       cin, cout, C.ptr(gw), C.stream_ptr())
        return gx, gw, None, None


def _module_tc_enabled():
    import os
    return os.environ.get('OSB_MODULE_TC', '1') != '0'


class _ConvBase(nn.Module):
    _osb_me_op = True      # an operator of this package (fast_eval.py looks for the module that CALLS them)
    TRANSPOSE = False

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
                 kernel_generator=None, expand_coordinates=False, convolution_mode=None, dimension=None):
        super().__init__()
        if dimension != 3:
            raise NotImplementedError("libosb200 implements 3-D sparse convolution (dimension=3)")
        if kernel_generator is not None or expand_coordinates:
            raise NotImplementedError("custom kernel generators / expand_coordinates are not on the OpenScene path")
        for name, v in (('kernel_size', kernel_size), ('stride', stride), ('dilation', dilation)):
            if not isinstance(v, int):
                if len(set(v)) != 1:
                    raise NotImplementedError(f"anisotropic {name} is not on the OpenScene path")
        ks = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = ks
        self.stride = stride if isinstance(stride, int) else stride[0]
        self.dilation = dilation if isinstance(dilation, int) else dilation[0]
        self.dimension = dimension
        self.kernel_volume = ks ** 3
        self.use_mm = self.kernel_volume == 1 and self.stride == 1
        shape = (in_channels, out_channels) if self.use_mm else (self.kernel_volume, in_channels, out_channels)
        self.kernel = nn.Parameter(torch.empty(*shape))
        self.bias = nn.Parameter(torch.empty(1, out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self, is_transpose=False):
        n = (self.out_channels if self.TRANSPOSE else self.in_channels) * self.kernel_volume
        stdv = 1.0 / math.sqrt(n)
        with torch.no_grad():
            self.kernel.uniform_(-stdv, stdv)
            if self.bias is not None:
                self.bias.uniform_(-stdv, stdv)

    def _w3(self):
        return self.kernel.unsqueeze(0) if self.kernel.dim() == 2 else self.kernel

    def _run_conv(self, input, kmap, n_out):
        """Inference (grad disabled) with channel counts that are multiples of 32 runs on the tensor-core kernel
        (bf16x3 split operands, ~1e-5 relative); everything else on the exact-fp32 kernels with autograd."""
        x = input._F
        K = self.kernel_volume if not self.use_mm else 1
        if (not torch.is_grad_enabled() and self.in_channels % 32 == 0 and self.out_channels % 32 == 0 and K <= 32
                and x.dtype == torch.float32 and _module_tc_enabled()):
            from . import tc
            key = (self.kernel.data_ptr(), self.kernel._version)
            if getattr(self, '_wpack_key', None) != key:
                self._wpack, self._wpack_key = tc.pack_weights(self._w3()), key
            xs = getattr(input, '_split', None)
            if xs is None:
                xs = tc.to_split(x)
                input._split = xs
            nbr = kmap.nbr if kmap is not None else None
            _, out = tc.conv_tc(xs, self.in_channels, None, 0, nbr, n_out, K, self._wpack, self.out_channels,
                                out_split=False, out_f32=True)
            return out
        return SparseConvFunction.apply(x, self._w3(), kmap, n_out)

    def __repr__(self):
        return (f"{self.__class__.__name__}(in={self.in_channels}, out={self.out_channels}, "
                f"kernel_size=[{self.kernel_size}]*3, stride=[{self.stride}]*3, dilation=[{self.dilation}]*3)")


class MinkowskiConvolution(_ConvBase):
    def forward(self, input):
        cm, ts = input.coordinate_manager, input._ts
        if self.use_mm:
            kmap, ts_out = None, ts
        else:
            ts_out = cm.stride(ts, self.stride) if self.stride > 1 else ts
            kmap = cm.kernel_map(ts, ts_out, self.kernel_size, self.dilation)
        n_out = cm.sets[ts_out].n
        out = self._run_conv(input, kmap, n_out)
        if self.bias is not None:
            out = out + self.bias
        return SparseTensor._wrap(out, cm, ts_out)


class MinkowskiConvolutionTranspose(_ConvBase):
    TRANSPOSE = True

    def forward(self, input):
        cm, ts = input.coordinate_manager, input._ts
        if ts % self.stride != 0 or (ts // self.stride) not in cm.sets:
            raise RuntimeError("MinkowskiConvolutionTranspose: the finer coordinate set must already exist "
                               "(U-Net decoder reuses the encoder's cached coordinates; SURVEY.md 8a a8)")
        ts_out = ts // self.stride
        if self.use_mm:
            kmap = None
        else:
            kmap = cm.kernel_map(ts_out, ts, self.kernel_size, self.dilation).transposed()
        n_out = cm.sets[ts_out].n
        out = self._run_conv(input, kmap, n_out)
        if self.bias is not None:
            out = out + self.bias
        return SparseTensor._wrap(out, cm, ts_out)


class MinkowskiBatchNorm(nn.Module):
    """Same structure as the reference stack: an ``nn.BatchNorm1d`` under ``.bn`` applied to the
    [N,C] feature matrix (resnet_base.py:79-80 touches ``m.bn.weight``).  The fused inference
    engine folds it into the convolution epilogue instead (openscene_b200/engine.py)."""
    _osb_me_op = True      # an operator of this package (fast_eval.py looks for the module that CALLS them)

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                 track_running_stats=track_running_stats)

    def forward(self, input):
        return SparseTensor._wrap(self.bn(input._F), input.coordinate_manager, input._ts)

    def __repr__(self):
        return f"MinkowskiBatchNorm({self.bn.num_features}, eps={self.bn.eps}, momentum={self.bn.momentum})"


class MinkowskiReLU(nn.Module):
    _osb_me_op = True      # an operator of this package (fast_eval.py looks for the module that CALLS them)
    def __init__(self, inplace=False):
        super().__init__()
        self.inplace = inplace

    def forward(self, input):
        return SparseTensor._wrap(torch.relu(input._F), input.coordinate_manager, input._ts)


class MinkowskiLinear(nn.Module):
    """``nn.Linear`` on the feature matrix.  A dense ``[B, C]`` tensor (what the global poolings return here) gives a dense
    tensor back, so ``final(glob_avg(x))`` of models/resnet_base.py:118-119 runs; a SparseTensor gives a SparseTensor."""
    _osb_me_op = True      # an operator of this package (fast_eval.py looks for the module that CALLS them)
    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.linear = nn.Linear(in_features, out_features, bias=bias)

    def forward(self, input):
        if isinstance(input, torch.Tensor):
            return self.linear(input)
        return SparseTensor._wrap(self.linear(input._F), input.coordinate_manager, input._ts)


# ------------------------------------------------------------------------------------------------
# pooling (csrc/pool.cu; the rules are DESIGN.md's "Pooling contract")
# ------------------------------------------------------------------------------------------------
POOL_SUM, POOL_AVG, POOL_MAX = 0, 1, 2


class SparsePoolFunction(torch.autograd.Function):
    """Sum / average / max over the kernel map ``kmap`` (nbr[K][n_out]); the backward walks ``kmap.transposed()``.
    Average pooling keeps the per-output count and max pooling the winning offset per (row, channel) for the backward."""

    @staticmethod
    def forward(ctx, x, kmap, mode):
        _require_f32(x, 'pooling input')
        if kmap.K > 65535:
            raise ValueError(f"openscene_b200: pooling supports kernel volumes up to 65535, got {kmap.K}")
        if x.shape[0] != kmap.n_in:
            raise ValueError(f"pooling input has {x.shape[0]} rows, its coordinate set has {kmap.n_in}")
        x = x.contiguous()
        c, n_out, dev = x.shape[1], kmap.n_out, x.device
        out = torch.empty((n_out, c), dtype=torch.float32, device=dev)
        count = torch.empty(n_out, dtype=torch.int32, device=dev) if mode == POOL_AVG else None
        argk = torch.empty((n_out, c), dtype=torch.int16, device=dev) if mode == POOL_MAX else None   # uint16 bits
        with torch.cuda.device(dev):
            C.call('osb_pool_fwd', C.ptr(x), c, C.ptr(kmap.nbr), n_out, kmap.K, mode, C.ptr(out), C.ptr(count),
                   C.ptr(argk), C.stream_ptr())
        ctx.kmap, ctx.mode = kmap, mode
        ctx.save_for_backward(count if mode == POOL_AVG else argk)
        return out

    @staticmethod
    def backward(ctx, g):
        _require_f32(g, 'pooling output gradient')
        (aux,) = ctx.saved_tensors
        g = g.contiguous()
        kt = ctx.kmap.transposed()
        gin = torch.empty((kt.n_out, g.shape[1]), dtype=torch.float32, device=g.device)
        count = aux if ctx.mode == POOL_AVG else None
        argk = aux if ctx.mode == POOL_MAX else None
        with torch.cuda.device(g.device):
            C.call('osb_pool_bwd', C.ptr(g), g.shape[1], C.ptr(kt.nbr), kt.n_out, kt.K, ctx.mode, C.ptr(count),
                   C.ptr(argk), C.ptr(gin), C.stream_ptr())
        return gin, None, None


class GlobalPoolFunction(torch.autograd.Function):
    """Sum / average / max of the rows of ``x`` per batch index ``batch`` (int32, one per row) -> dense [n_batch, C]."""

    @staticmethod
    def forward(ctx, x, batch, n_batch, mode):
        _require_f32(x, 'global pooling input')
        x = x.contiguous()
        n, c, dev = x.shape[0], x.shape[1], x.device
        out = torch.empty((n_batch, c), dtype=torch.float32, device=dev)
        count = torch.empty(n_batch, dtype=torch.int32, device=dev) if mode == POOL_AVG else None
        argrow = torch.empty((n_batch, c), dtype=torch.int32, device=dev) if mode == POOL_MAX else None
        ws_bytes = C.lib().osb_global_pool_workspace_bytes(n, c, n_batch)
        with torch.cuda.device(dev):
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            C.call('osb_global_pool_fwd', C.ptr(x), C.ptr(batch), n, c, n_batch, mode, C.ptr(out), C.ptr(count),
                   C.ptr(argrow), C.ptr(ws), ws_bytes, C.stream_ptr())
        ctx.mode, ctx.n = mode, n
        ctx.save_for_backward(batch, count if mode == POOL_AVG else argrow)
        return out

    @staticmethod
    def backward(ctx, g):
        _require_f32(g, 'global pooling output gradient')
        batch, aux = ctx.saved_tensors
        g = g.contiguous()
        gin = torch.empty((ctx.n, g.shape[1]), dtype=torch.float32, device=g.device)
        count = aux if ctx.mode == POOL_AVG else None
        argrow = aux if ctx.mode == POOL_MAX else None
        with torch.cuda.device(g.device):
            C.call('osb_global_pool_bwd', C.ptr(g), C.ptr(batch), ctx.n, g.shape[1], ctx.mode, C.ptr(count), C.ptr(argrow),
                   C.ptr(gin), C.stream_ptr())
        return gin, None, None, None


class _PoolBase(nn.Module):
    _osb_me_op = True      # an operator of this package (fast_eval.py looks for the module that CALLS them)
    MODE = None

    def __init__(self, kernel_size, stride=1, dilation=1, kernel_generator=None, dimension=None):
        super().__init__()
        if dimension != 3:
            raise NotImplementedError("dimension=3 only")
        if kernel_generator is not None:
            raise NotImplementedError("custom kernel generators are not implemented")
        for name, v in (('kernel_size', kernel_size), ('stride', stride), ('dilation', dilation)):
            if not isinstance(v, int) and len(set(v)) != 1:
                raise NotImplementedError(f"anisotropic {name} is not implemented")
        self.kernel_size = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
        self.stride = stride if isinstance(stride, int) else stride[0]
        self.dilation = dilation if isinstance(dilation, int) else dilation[0]

    def forward(self, input):
        cm, ts = input.coordinate_manager, input._ts
        ts_out = cm.stride(ts, self.stride) if self.stride > 1 else ts
        kmap = cm.kernel_map(ts, ts_out, self.kernel_size, self.dilation)
        return SparseTensor._wrap(SparsePoolFunction.apply(input._F, kmap, self.MODE), cm, ts_out)

    def __repr__(self):
        return (f"{self.__class__.__name__}(kernel_size=[{self.kernel_size}]*3, stride=[{self.stride}]*3, "
                f"dilation=[{self.dilation}]*3)")


class MinkowskiSumPooling(_PoolBase):
    """Sum over the inputs present in the window (fp32 adds in offset order)."""
    MODE = POOL_SUM


class MinkowskiAvgPooling(_PoolBase):
    """Sum over the present inputs divided by their count (an output with none gives 0)."""
    MODE = POOL_AVG


class MinkowskiMaxPooling(_PoolBase):
    """Per channel the largest present input: the first NaN in offset order wins, ties go to the lowest offset and an output
    with no present input gives 0 and receives no gradient."""
    MODE = POOL_MAX


class _GlobalPoolBase(nn.Module):
    """Pooling over all rows of each batch index, in ``.F`` row order.  Returns the dense ``[B, C]`` matrix with
    ``B = max batch index + 1`` (MinkowskiEngine returns a SparseTensor whose ``.F`` is this matrix); a batch index without
    rows gives 0 (sum), NaN (average) or -inf (max)."""
    _osb_me_op = True      # an operator of this package (fast_eval.py looks for the module that CALLS them)
    MODE = None

    def __init__(self, dimension=None, **kw):
        super().__init__()

    def forward(self, input):
        batch, n_batch = input.coordinate_manager.batch_index(input._ts)
        return GlobalPoolFunction.apply(input.F, batch, n_batch, self.MODE)


class MinkowskiGlobalSumPooling(_GlobalPoolBase):
    MODE = POOL_SUM


class MinkowskiGlobalAvgPooling(_GlobalPoolBase):
    MODE = POOL_AVG


class MinkowskiGlobalMaxPooling(_GlobalPoolBase):
    MODE = POOL_MAX
