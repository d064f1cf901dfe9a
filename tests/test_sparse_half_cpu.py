"""The half-precision sparse convolution without a GPU: argument validation of its C entry points before any CUDA call,
its workspace-size queries, the feature losses' rejection of the bf16 dtype code, and the feature dtypes SparseTensor
accepts."""
import ctypes as C

import pytest
import torch

from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200 import sparse as sp

F16, BF16, F32 = _lib.FEAT_F16, _lib.FEAT_BF16, _lib.FEAT_F32


def _off(*v):
    return (C.c_int64 * len(v))(*v)


def _fwd(l, dtype=BF16, K=1, off=None, pairs=16, n_in=4, ci=3, x=16, w=16, n_out=4, co=3, ws=16, out=16):
    return l.sgb_sparse_conv_half_forward(dtype, K, _off(0, 2) if off is None else off, pairs, 0, n_in, ci, x, w,
                                          n_out, co, ws, out, None)


def _bwd_in(l, dtype=F16, K=1, off=None, pairs=16, dx=16, w=16, dy=16, ws=16):
    return l.sgb_sparse_conv_half_backward_input(dtype, K, _off(0, 2) if off is None else off, pairs, 1, 4, 3, dx, w,
                                                 4, 3, dy, ws, None)


def _bwd_w(l, dtype=BF16, K=1, off=None, pairs=16, x=16, dy=16, ws=16, dW=16):
    return l.sgb_sparse_conv_half_backward_weight(dtype, K, _off(0, 2) if off is None else off, pairs, 0, 4, 3, x, 4,
                                                  3, dy, ws, dW, None)


@pytest.mark.parametrize("call,msg", [
    (lambda l: _fwd(l, dtype=F32), b"dtype 1"),
    (lambda l: _fwd(l, dtype=7), b"dtype 7"),
    (lambda l: _bwd_in(l, dtype=-1), b"dtype -1"),
    (lambda l: _bwd_w(l, dtype=F32), b"dtype 1"),
    (lambda l: _fwd(l, K=0, off=_off(0)), b"K = 0"),
    (lambda l: _fwd(l, K=126, off=_off(*[0] * 127)), b"K = 126"),
    (lambda l: _bwd_in(l, K=200), b"K = 200"),
    (lambda l: _bwd_w(l, K=0, off=_off(0)), b"K = 0"),
    (lambda l: _fwd(l, ci=0), b"C_in = 0"),
    (lambda l: _fwd(l, co=-1), b"C_out = -1"),
    (lambda l: _fwd(l, off=C.cast(None, C.POINTER(C.c_int64))), b"null offsets"),
    (lambda l: _fwd(l, K=2, off=_off(0, 3, 2)), b"decrease"),
    (lambda l: _bwd_w(l, K=2, off=_off(1, 3, 4)), b"offsets[0] = 1"),
    (lambda l: _fwd(l, n_in=-1), b"row counts"),
    (lambda l: _fwd(l, n_out=2 ** 31), b"row counts"),
    (lambda l: _fwd(l, pairs=None), b"pairs"),
    (lambda l: _fwd(l, pairs=20), b"unaligned pairs"),
    (lambda l: _fwd(l, x=None), b"null x"),
    (lambda l: _fwd(l, w=None), b"null x / kernel / out"),
    (lambda l: _fwd(l, out=None), b"null x / kernel / out"),
    (lambda l: _fwd(l, ws=None), b"workspace"),
    (lambda l: _fwd(l, ws=24), b"unaligned workspace"),
    (lambda l: _bwd_in(l, dx=None), b"null dx"),
    (lambda l: _bwd_in(l, dy=None), b"null dx / kernel / dy"),
    (lambda l: _bwd_in(l, ws=None), b"workspace"),
    (lambda l: _bwd_w(l, x=None), b"null x"),
    (lambda l: _bwd_w(l, dW=None), b"null x / dy / dkernel"),
    (lambda l: _bwd_w(l, ws=8), b"unaligned workspace"),
])
def test_half_entry_points_validate_before_cuda(call, msg):
    lib = _lib.load()
    assert call(lib) == -1
    assert msg in lib.sgb_last_error()


def test_half_workspace_queries_reject_what_the_calls_reject():
    lib = _lib.load()
    for q in (lib.sgb_sparse_conv_half_forward_workspace_bytes,
              lib.sgb_sparse_conv_half_backward_input_workspace_bytes):
        assert q(BF16, 1, _off(0, 5), 10, 3, 20, 7) > 0
        assert q(F32, 1, _off(0, 5), 10, 3, 20, 7) == 0
        assert q(BF16, 0, _off(0), 10, 3, 20, 7) == 0
        assert q(F16, 1, _off(0, 5), 10, 0, 20, 7) == 0
        assert q(F16, 2, _off(0, 5, 4), 10, 3, 20, 7) == 0
        assert q(F16, 1, _off(0, 5), -1, 3, 20, 7) == 0
    # one fp32 copy of out (forward) or dx (input gradient)
    assert lib.sgb_sparse_conv_half_forward_workspace_bytes(F16, 1, _off(0, 5), 10, 3, 1000, 70) >= 4 * 1000 * 70
    assert lib.sgb_sparse_conv_half_backward_input_workspace_bytes(F16, 1, _off(0, 5), 1000, 70, 10, 3) >= 4 * 1000 * 70
    w = lib.sgb_sparse_conv_half_backward_weight_workspace_bytes
    assert w(BF16, 2, _off(0, 5000, 5001), 3, 7) == lib.sgb_sparse_conv_backward_weight_workspace_bytes(
        2, _off(0, 5000, 5001), 3, 7) >= 4 * 4 * 3 * 7
    assert w(F32, 1, _off(0, 5), 3, 3) == 0 and w(BF16, 0, _off(0), 3, 3) == 0 and w(F16, 1, _off(0, 5), 3, 0) == 0


def test_feature_losses_reject_the_bf16_code():
    lib = _lib.load()
    assert lib.sgb_feature_map_loss(8, 10, 16, 16, BF16, 0, 16, 16, None) == -1
    assert b"target_dtype 2" in lib.sgb_last_error()
    assert lib.sgb_voxel_feature_loss(10, 8, 16, 16, 10, 8, 0, 16, BF16, 0, 16, 16, 16, None) == -1
    assert b"target_dtype 2" in lib.sgb_last_error()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32, torch.float64])
def test_sparse_tensor_still_needs_cuda_features(dtype):
    with pytest.raises(ValueError, match="float32 CUDA"):
        sp.SparseTensor(torch.zeros(4, 3, dtype=dtype), torch.zeros(4, 4, dtype=torch.int32))
