"""The expected-depth / alpha entry points without a GPU: the symbols are bound, and the requests the library
refuses (C > 4, half of the forward outputs, CPU tensors) are refused during argument checking, before any ctx is
used or anything is enqueued."""
import ctypes as C

import pytest
import torch

from semantic_gaussians_b200 import _lib

E_INVALID = -1   # SGB_E_INVALID, include/sgb200.h


def _inputs(**kw):
    base = dict(P=10, D=0, M=0, W=64, H=64, C=3, background=1, means3D=1, shs=None, colors_precomp=1, opacities=1,
                scales=1, scale_modifier=1.0, rotations=1, cov3D_precomp=None, viewmatrix=1, projmatrix=1, campos=1,
                tan_fovx=0.5, tan_fovy=0.5, prefiltered=0, debug=0)
    base.update(kw)
    return _lib.ViewInputs(**base)


def test_new_symbols_are_bound():
    lib = _lib.load()
    for name in ("sgb_forward_render_batch_ext", "sgb_backward_batch_ext"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert getattr(lib, name).argtypes is not None


def _forward_ext(C_, exp, alpha):
    lib = _lib.load()
    cams = _lib.Camera(1, 1, 1, 0.5, 0.5)
    one = C.c_void_p(1)
    R = (C.c_int64 * 1)(1)
    # ctx 1 is a dummy: the call must fail before it is dereferenced
    return lib.sgb_forward_render_batch_ext(1, C.byref(_inputs(C=C_)), 1, C.byref(cams), R, one, one, one, one, one,
                                            None, exp, alpha, None)


@pytest.mark.parametrize("C_", [5, 16, 256])
def test_wide_rasters_refuse_expected_depth_and_alpha(C_):
    lib = _lib.load()
    one = C.c_void_p(1)
    assert _forward_ext(C_, one, one) == E_INVALID
    assert b"C <= 4" in lib.sgb_last_error()
    cams = _lib.Camera(1, 1, 1, 0.5, 0.5)
    grads = _lib.ViewGrads(*[1] * 9)
    R = (C.c_int64 * 1)(1)
    for exp, alpha in ((one, None), (None, one), (one, one)):
        rc = lib.sgb_backward_batch_ext(1, C.byref(_inputs(C=C_)), 1, C.byref(cams), R, one, one, one, one, one,
                                        exp, alpha, C.byref(grads), None)
        assert rc == E_INVALID and b"C <= 4" in lib.sgb_last_error()


def test_expected_depth_and_alpha_come_together():
    lib = _lib.load()
    one = C.c_void_p(1)
    for exp, alpha in ((one, None), (None, one)):
        assert _forward_ext(3, exp, alpha) == E_INVALID
        assert b"together" in lib.sgb_last_error()


def test_cpu_tensors_are_rejected():
    from semantic_gaussians_b200 import rgbd_rasterization as rgbd
    rs = rgbd.GaussianRasterizationSettings(8, 8, 1.0, 1.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                            torch.zeros(3), False, False)
    z = torch.zeros
    with pytest.raises(RuntimeError, match="no CPU path"):
        rgbd.GaussianRasterizer(rs).forward_expected_depth(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1),
                                                           colors_precomp=z(1, 3), scales=z(1, 3), rotations=z(1, 4))
