"""Sparse 3D convolution on the GPU: the parts of MinkowskiEngine (ME) that the reference's MinkUNet uses.

``SparseTensor(features, coordinates)`` takes ME's positional order and has ``.F``, ``.C`` and ``.tensor_stride``.
Its ``CoordinateManager`` caches, for the tensors derived from one input (one forward), the coordinate map of each
tensor stride and the kernel map of each ``(in stride, out stride, kernel size)``: the BasicBlocks at one stride
share their 3x3x3 map, and each transposed layer reuses the pairs of the stride-2 layer it mirrors.

Coordinates are int32 rows ``(b, x, y, z)``.  Duplicate rows and negative x, y, z raise ``ValueError``.  Host reads:
one for the input map (its duplicate / negative counts), one per strided map (its row count) and one per kernel map
(its per-offset pair counts).  The convolution products never synchronise.

Layers: ``Convolution`` (``kernel`` shaped ``(K, in, out)``, or ``(in, out)`` for kernel size 1, no bias),
``ConvolutionTranspose``, ``BatchNorm`` (``.bn`` is a ``torch.nn.BatchNorm1d``), ``ReLU`` and ``cat``.  Supported:
kernel size 3 or 5 at stride 1, kernel size 1 at stride 1 (a dense ``torch.mm``), kernel size 2 at stride 2, forward
and transposed; anything else, dilation != 1 and D != 3 raise ``NotImplementedError``.

Features are CUDA float32, float16 or bfloat16.  Under ``torch.autocast("cuda")`` a layer runs its product in the
autocast dtype; outside it, the features' own dtype decides.  fp16 / bf16 products run on tensor cores: each output
element is accumulated in fp32 over every offset and rounded once, and the kernel parameter stays fp32 (it is rounded
to the half type once per forward, and its gradient is accumulated and returned in fp32).

Offsets (sgb200.h): index d = jx + k jy + k^2 jz, offset lb + j t per axis with lb = -((k-1)//2) t for odd k and 0
for k = 2.  This is how we read ME's hyper-cube region; it has not been compared with ME itself."""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from . import _lib

_SUPPORTED = {(1, 1), (3, 1), (5, 1), (2, 2)}   # (kernel size, stride)


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


_HALF = {torch.float16: _lib.FEAT_F16, torch.bfloat16: _lib.FEAT_BF16}


def _check_features(F, what="features"):
    if not isinstance(F, torch.Tensor) or not F.is_cuda or F.dtype not in (torch.float32, *_HALF) or F.dim() != 2:
        desc = f"{tuple(F.shape)} {F.dtype} on {F.device}" if isinstance(F, torch.Tensor) else type(F).__name__
        raise ValueError(f"{what} must be a 2-D float32 CUDA tensor (or float16 / bfloat16), got {desc}")


def _product_dtype(F):
    """The dtype a layer computes in: the autocast dtype under torch.autocast("cuda"), else the features' own."""
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        return dt if dt in _HALF else torch.float32
    return F.dtype


class CoordinateMap:
    """The rows of one tensor stride and their device hash table."""

    def __init__(self, coords: torch.Tensor, stride: int):
        self.coords, self.stride, self.n = coords, stride, coords.shape[0]
        lib = _lib.load()
        self.table = torch.empty(lib.sgb_coord_map_bytes(self.n), dtype=torch.uint8, device=coords.device)
        self.status = torch.empty(2, dtype=torch.int64, device=coords.device)
        _lib.check(lib.sgb_coord_map_build(self.n, coords.data_ptr(), self.table.data_ptr(), self.status.data_ptr(),
                                           _stream(coords.device)), "sgb_coord_map_build")


class KernelMap:
    """(in row, out row) int32 pairs of every kernel offset, and the host copy of the per-offset offsets."""

    def __init__(self, in_map: CoordinateMap, out_map: CoordinateMap, k: int):
        lib = _lib.load()
        dev = in_map.coords.device
        self.K = k ** 3
        s = _stream(dev)
        ws = torch.empty(lib.sgb_kernel_map_workspace_bytes(out_map.n, k), dtype=torch.uint8, device=dev)
        offsets = torch.empty(self.K + 1, dtype=torch.int64, device=dev)
        args = (in_map.n, in_map.coords.data_ptr(), in_map.table.data_ptr(), out_map.n, out_map.coords.data_ptr(), k,
                in_map.stride, ws.data_ptr())
        _lib.check(lib.sgb_kernel_map_count(*args, offsets.data_ptr(), s), "sgb_kernel_map_count")
        off = offsets.tolist()                                             # the one host read of this map
        self.offsets_host = (C.c_int64 * (self.K + 1))(*off)
        self.pairs = torch.empty((max(off[-1], 1), 2), dtype=torch.int32, device=dev)
        if off[-1]:
            _lib.check(lib.sgb_kernel_map_fill(*args, self.pairs.data_ptr(), s), "sgb_kernel_map_fill")
        self.pairs = self.pairs[:off[-1]]
        self.counts = [b - a for a, b in zip(off[:-1], off[1:])]


class CoordinateManager:
    """Coordinate maps by tensor stride and kernel maps by (in stride, out stride, k), built on first use."""

    def __init__(self, coordinates: torch.Tensor):
        if not isinstance(coordinates, torch.Tensor) or not coordinates.is_cuda:
            raise ValueError("coordinates must be a CUDA tensor")
        if coordinates.dim() != 2 or coordinates.shape[1] != 4 or coordinates.shape[0] == 0:
            raise ValueError(f"coordinates must be (N, 4) rows (b, x, y, z) with N > 0, got {tuple(coordinates.shape)}")
        if coordinates.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"coordinates must be int32 or int64, got {coordinates.dtype}")
        if coordinates.dtype == torch.int64:
            if coordinates.abs().max().item() >= 2 ** 31:
                raise ValueError("coordinates do not fit in int32")
        coords = torch.empty(coordinates.shape, dtype=torch.int32, device=coordinates.device)
        coords.copy_(coordinates)                         # own, contiguous, 16-byte aligned rows
        m = CoordinateMap(coords, 1)
        dup, neg = m.status.tolist()
        if neg:
            raise ValueError(f"{neg} coordinate rows have a negative x, y or z")
        if dup:
            raise ValueError(f"{dup} coordinate rows repeat an earlier row; quantize the input first")
        self.device = coordinates.device
        self.maps = {1: m}
        self.kernel_maps = {}

    def map(self, stride: int) -> CoordinateMap:
        m = self.maps.get(stride)
        if m is None:
            if stride < 2 or stride & (stride - 1):
                raise ValueError(f"no coordinate map at tensor stride {stride}")
            src = self.map(stride // 2)
            lib = _lib.load()
            ws = torch.empty(lib.sgb_coord_stride_workspace_bytes(src.n), dtype=torch.uint8, device=self.device)
            out = torch.empty((src.n, 4), dtype=torch.int32, device=self.device)
            count = torch.empty(1, dtype=torch.int64, device=self.device)
            _lib.check(lib.sgb_coord_stride(src.n, src.coords.data_ptr(), src.stride, ws.data_ptr(), out.data_ptr(),
                                            count.data_ptr(), _stream(self.device)), "sgb_coord_stride")
            n = int(count.item())                                          # the one host read of this map
            m = self.maps[stride] = CoordinateMap(out[:n], stride)
        return m

    def kernel_map(self, in_stride: int, out_stride: int, k: int) -> KernelMap:
        key = (in_stride, out_stride, k)
        km = self.kernel_maps.get(key)
        if km is None:
            km = self.kernel_maps[key] = KernelMap(self.map(in_stride), self.map(out_stride), k)
        return km


class SparseTensor:
    """Features ``F`` (N, C) on the rows ``C`` (N, 4) of one tensor stride of a coordinate manager."""

    def __init__(self, features, coordinates=None, tensor_stride=1, coordinate_manager=None):
        _check_features(features)
        if coordinate_manager is None:
            if coordinates is None:
                raise ValueError("SparseTensor needs coordinates or a coordinate manager")
            coordinate_manager = CoordinateManager(coordinates)
        if isinstance(tensor_stride, (list, tuple)):
            if len(set(tensor_stride)) != 1:
                raise NotImplementedError("only equal tensor strides on every axis are supported")
            tensor_stride = tensor_stride[0]
        self.coordinate_manager = coordinate_manager
        self._stride = int(tensor_stride)
        n = coordinate_manager.map(self._stride).n
        if features.shape[0] != n:
            raise ValueError(f"features have {features.shape[0]} rows, the coordinate map {n}")
        self.F = features

    @property
    def C(self) -> torch.Tensor:
        return self.coordinate_manager.map(self._stride).coords

    @property
    def tensor_stride(self):
        return [self._stride] * 3

    def _same_map(self, other, what):
        if other.coordinate_manager is not self.coordinate_manager or other._stride != self._stride:
            raise ValueError(f"{what} needs both tensors on the same coordinate map")

    def _with(self, features):
        return SparseTensor(features, tensor_stride=self._stride, coordinate_manager=self.coordinate_manager)

    def __add__(self, other):
        self._same_map(other, "+")
        return self._with(self.F + other.F)


class _SparseConvFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, kernel, kmap, transposed, n_out):
        lib = _lib.load()
        x, kernel = x.contiguous(), kernel.contiguous()
        out = torch.empty((n_out, kernel.shape[2]), dtype=torch.float32, device=x.device)
        _lib.check(lib.sgb_sparse_conv_forward(kmap.K, kmap.offsets_host, kmap.pairs.data_ptr(), int(transposed),
                                               x.shape[0], x.shape[1], x.data_ptr(), kernel.data_ptr(), n_out,
                                               kernel.shape[2], out.data_ptr(), _stream(x.device)),
                   "sgb_sparse_conv_forward")
        ctx.save_for_backward(x, kernel)
        ctx.kmap, ctx.transposed = kmap, int(transposed)
        return out

    @staticmethod
    def backward(ctx, dy):
        lib = _lib.load()
        x, kernel = ctx.saved_tensors
        km, dy = ctx.kmap, dy.contiguous()
        K, Ci, Co = kernel.shape
        s = _stream(x.device)
        dx = dW = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _lib.check(lib.sgb_sparse_conv_backward_input(K, km.offsets_host, km.pairs.data_ptr(), ctx.transposed,
                                                          x.shape[0], Ci, dx.data_ptr(), kernel.data_ptr(),
                                                          dy.shape[0], Co, dy.data_ptr(), s),
                       "sgb_sparse_conv_backward_input")
        if ctx.needs_input_grad[1]:
            dW = torch.empty_like(kernel)
            nbytes = lib.sgb_sparse_conv_backward_weight_workspace_bytes(K, km.offsets_host, Ci, Co)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            _lib.check(lib.sgb_sparse_conv_backward_weight(K, km.offsets_host, km.pairs.data_ptr(), ctx.transposed,
                                                           x.shape[0], Ci, x.data_ptr(), dy.shape[0], Co,
                                                           dy.data_ptr(), ws.data_ptr(), dW.data_ptr(), s),
                       "sgb_sparse_conv_backward_weight")
        return dx, dW, None, None, None


class _HalfSparseConvFunction(torch.autograd.Function):
    """The product on fp16 / bf16 features x with the fp32 kernel parameter: the kernel is rounded to x's dtype once
    here, that copy is saved for the input gradient, and the kernel gradient is the fp32 one of the native call."""

    @staticmethod
    def forward(ctx, x, kernel, kmap, transposed, n_out):
        lib = _lib.load()
        dtype = _HALF[x.dtype]
        x, wh = x.contiguous(), kernel.detach().to(x.dtype).contiguous()
        K, Ci, Co = wh.shape
        out = torch.empty((n_out, Co), dtype=x.dtype, device=x.device)
        nbytes = lib.sgb_sparse_conv_half_forward_workspace_bytes(dtype, K, kmap.offsets_host, x.shape[0], Ci, n_out,
                                                                  Co)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        _lib.check(lib.sgb_sparse_conv_half_forward(dtype, K, kmap.offsets_host, kmap.pairs.data_ptr(), int(transposed),
                                                    x.shape[0], Ci, x.data_ptr(), wh.data_ptr(), n_out, Co,
                                                    ws.data_ptr(), out.data_ptr(), _stream(x.device)),
                   "sgb_sparse_conv_half_forward")
        ctx.save_for_backward(x, wh)
        ctx.kmap, ctx.transposed = kmap, int(transposed)
        return out

    @staticmethod
    def backward(ctx, dy):
        lib = _lib.load()
        x, wh = ctx.saved_tensors
        km, dy = ctx.kmap, dy.to(x.dtype).contiguous()
        dtype = _HALF[x.dtype]
        K, Ci, Co = wh.shape
        s = _stream(x.device)
        dx = dW = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            nbytes = lib.sgb_sparse_conv_half_backward_input_workspace_bytes(dtype, K, km.offsets_host, x.shape[0], Ci,
                                                                             dy.shape[0], Co)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            _lib.check(lib.sgb_sparse_conv_half_backward_input(dtype, K, km.offsets_host, km.pairs.data_ptr(),
                                                               ctx.transposed, x.shape[0], Ci, dx.data_ptr(),
                                                               wh.data_ptr(), dy.shape[0], Co, dy.data_ptr(),
                                                               ws.data_ptr(), s),
                       "sgb_sparse_conv_half_backward_input")
        if ctx.needs_input_grad[1]:
            dW = torch.empty(wh.shape, dtype=torch.float32, device=x.device)
            nbytes = lib.sgb_sparse_conv_half_backward_weight_workspace_bytes(dtype, K, km.offsets_host, Ci, Co)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            _lib.check(lib.sgb_sparse_conv_half_backward_weight(dtype, K, km.offsets_host, km.pairs.data_ptr(),
                                                                ctx.transposed, x.shape[0], Ci, x.data_ptr(),
                                                                dy.shape[0], Co, dy.data_ptr(), ws.data_ptr(),
                                                                dW.data_ptr(), s),
                       "sgb_sparse_conv_half_backward_weight")
        return dx, dW, None, None, None


def _check_layer(kernel_size, stride, dilation, dimension, transposed):
    if dimension != 3:
        raise NotImplementedError(f"dimension {dimension}: only D = 3 is supported")
    if dilation != 1:
        raise NotImplementedError(f"dilation {dilation}: only 1 is supported")
    if transposed and (kernel_size, stride) != (2, 2):
        raise NotImplementedError(f"transposed kernel_size={kernel_size}, stride={stride}: only 2, 2 is supported")
    if (kernel_size, stride) not in _SUPPORTED:
        raise NotImplementedError(f"kernel_size={kernel_size}, stride={stride}: supported are k = 3 or 5 and k = 1 "
                                  "at stride 1, and k = 2 at stride 2")


class _ConvBase(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride, dilation, bias, dimension, transposed):
        super().__init__()
        _check_layer(kernel_size, stride, dilation, dimension, transposed)
        if bias:
            raise NotImplementedError("bias is not supported")
        if in_channels <= 0 or out_channels <= 0:
            raise ValueError(f"channel counts must be positive, got {in_channels}, {out_channels}")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.is_transpose = kernel_size, stride, transposed
        K = kernel_size ** 3
        shape = (K, in_channels, out_channels) if K > 1 else (in_channels, out_channels)
        self.kernel = nn.Parameter(torch.empty(shape))
        # ME's reset_parameters: uniform in +-1/sqrt(fan), fan = (out if transposed else in) channels * K
        bound = 1.0 / math.sqrt((out_channels if transposed else in_channels) * K)
        with torch.no_grad():
            self.kernel.uniform_(-bound, bound)

    def _product(self, x: SparseTensor, kmap, transposed, out_stride):
        _check_features(x.F, "input features")
        if x.F.shape[1] != self.in_channels:
            raise ValueError(f"input has {x.F.shape[1]} channels, the layer {self.in_channels}")
        n_out = x.coordinate_manager.map(out_stride).n
        dt = _product_dtype(x.F)
        if dt == torch.float32:
            F = _SparseConvFunction.apply(x.F.float(), self.kernel, kmap, transposed, n_out)
        else:
            F = _HalfSparseConvFunction.apply(x.F.to(dt), self.kernel, kmap, transposed, n_out)
        return SparseTensor(F, tensor_stride=out_stride, coordinate_manager=x.coordinate_manager)


class Convolution(_ConvBase):
    """ME.MinkowskiConvolution for kernel_size 3 / 5 / 1 at stride 1 and 2 at stride 2."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, dilation=1, bias=False, dimension=3):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, bias, dimension, False)

    def forward(self, x: SparseTensor) -> SparseTensor:
        t = x._stride
        if self.kernel_size == 1:
            _check_features(x.F, "input features")
            dt = _product_dtype(x.F)
            return x._with(torch.mm(x.F.to(dt), self.kernel.to(dt)))
        km = x.coordinate_manager.kernel_map(t, t * self.stride, self.kernel_size)
        return self._product(x, km, False, t * self.stride)


class ConvolutionTranspose(_ConvBase):
    """ME.MinkowskiConvolutionTranspose for kernel_size 2, stride 2: writes onto the existing finer map."""

    def __init__(self, in_channels, out_channels, kernel_size=2, stride=2, dilation=1, bias=False, dimension=3):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, bias, dimension, True)

    def forward(self, x: SparseTensor) -> SparseTensor:
        t = x._stride
        if t < 2 or (t // 2) not in x.coordinate_manager.maps:
            raise ValueError(f"transposed layer at tensor stride {t}: no finer map to write onto")
        km = x.coordinate_manager.kernel_map(t // 2, t, 2)
        return self._product(x, km, True, t // 2)


class BatchNorm(nn.Module):
    """ME.MinkowskiBatchNorm: torch.nn.BatchNorm1d over the rows, as ``.bn``."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                 track_running_stats=track_running_stats)

    def forward(self, x: SparseTensor) -> SparseTensor:
        return x._with(self.bn(x.F))


class ReLU(nn.Module):
    def __init__(self, inplace=False):
        super().__init__()

    def forward(self, x: SparseTensor) -> SparseTensor:
        return x._with(torch.relu(x.F))


def cat(*tensors: SparseTensor) -> SparseTensor:
    """Channels of tensors on one coordinate map, concatenated in argument order."""
    for t in tensors[1:]:
        tensors[0]._same_map(t, "cat")
    return tensors[0]._with(torch.cat([t.F for t in tensors], dim=1))
