"""Photometric loss without a GPU: the numpy oracle (value and analytic gradient) against torch float64 autograd
of the reference's expressions, argument validation of the two C entry points (before any CUDA call), and the
Python layer's ValueErrors."""
import ctypes as C

import numpy as np
import pytest
import torch

from loss_ref import photometric_torch, ssim_torch, taps_fp32, window
from oracle import loss_oracle as lo
from semantic_gaussians_b200 import _lib


def _pair(shape, seed, ties=0.0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 1, shape)
    y = rng.uniform(0, 1, shape)
    if ties:
        tie = rng.uniform(0, 1, shape) < ties
        y[tie] = x[tie]          # |x - y| has a kink here: abs()'s backward gives sign(0) = 0
    return x, y


def _torch_loss_and_grad(x, y, lam, cut_edge):
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    yt = torch.tensor(y, dtype=torch.float64)
    loss, l1 = photometric_torch(xt, yt, window(torch.float64, separable_fp64=True), lam, cut_edge)
    loss.backward()
    return float(loss.detach()), float(l1.detach()), xt.grad.numpy()


def test_window_taps_match_the_reference_construction():
    np.testing.assert_array_equal(lo.window_taps(), taps_fp32().numpy())
    assert abs(float(lo.window_taps().astype(np.float64).sum()) - 1.0) < 1e-6


@pytest.mark.parametrize("shape,cut_edge,lam,ties", [
    ((3, 13, 17), False, 0.2, 0.3),       # small planes with tied pixels
    ((3, 11, 11), False, 0.5, 0.0),       # exactly one window
    ((1, 5, 7), False, 0.2, 0.2),         # smaller than the window
    ((2, 5, 7), False, 1.0, 0.0),         # pure D-SSIM
    ((3, 104, 203), True, 0.2, 0.1),      # border crop h//100 = 1, w//100 = 2
    ((2, 3, 16, 20), False, 0.2, 0.1),    # (N,C,H,W)
])
def test_oracle_matches_torch_float64_autograd(shape, cut_edge, lam, ties):
    x, y = _pair(shape, seed=sum(shape), ties=ties)
    want_loss, want_l1, want_g = _torch_loss_and_grad(x, y, lam, cut_edge)
    loss, l1, g = lo.photometric_loss(x, y, lam, cut_edge)
    assert abs(loss - want_loss) <= 1e-13
    assert abs(l1 - want_l1) <= 1e-13
    scale = np.abs(want_g).max()
    assert np.abs(g - want_g).max() <= 1e-11 * scale, np.abs(g - want_g).max() / scale
    if cut_edge:
        h, w = shape[-2:]
        assert not g[..., : h // 100, :].any() and not g[..., :, w - w // 100:].any()


def test_oracle_ssim_matches_torch_float64_autograd():
    x, y = _pair((2, 3, 9, 14), seed=5)
    xt = torch.tensor(x, requires_grad=True)
    s = ssim_torch(xt, torch.tensor(y), window(torch.float64, separable_fp64=True))
    s.backward()
    val, g = lo.ssim(x, y)
    assert abs(val - float(s)) <= 1e-13
    assert np.abs(g - xt.grad.numpy()).max() <= 1e-11 * np.abs(g).max()


def test_identical_images_have_unit_ssim_and_zero_loss():
    x, _ = _pair((3, 20, 24), seed=1)
    loss, l1, g = lo.photometric_loss(x, x, 0.2)
    assert abs(loss) < 1e-12 and l1 == 0.0
    assert np.abs(g).max() < 1e-9


# ---- C entry points: argument validation before any CUDA call (no GPU here)

def _fwd(lib, planes=3, h=8, w=8, x=1, xps=64, xrs=8, y=1, yps=64, yrs=8, sums=1, partials=None):
    return lib.sgb_photometric_forward(planes, h, w, x, xps, xrs, y, yps, yrs, sums, partials, None)


def _bwd(lib, planes=3, h=8, w=8, x=1, xps=64, xrs=8, y=1, yps=64, yrs=8, partials=1, coef=1, dx=1, dps=64, drs=8):
    return lib.sgb_photometric_backward(planes, h, w, x, xps, xrs, y, yps, yrs, partials, coef, dx, dps, drs, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(planes=0), b"need planes > 0, h > 0, w > 0"),
    (dict(h=0), b"need planes > 0, h > 0, w > 0"),
    (dict(w=-3), b"need planes > 0, h > 0, w > 0"),
    (dict(h=65535 * 32 + 1), b"exceeds"),
    (dict(x=None), b"null x, y or sums"),
    (dict(sums=None), b"null x, y or sums"),
    (dict(xrs=7), b"x: row stride smaller than the row"),
    (dict(yps=63), b"y: plane stride smaller than the plane"),
    (dict(xrs=-8), b"x: row stride"),
])
def test_forward_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _fwd(lib, **kw) == -1
    assert msg in lib.sgb_last_error()


@pytest.mark.parametrize("kw,msg", [
    (dict(planes=-1), b"need planes > 0, h > 0, w > 0"),
    (dict(partials=None), b"null x, y, partials, coef or dL_dx"),
    (dict(coef=None), b"null x, y, partials, coef or dL_dx"),
    (dict(dx=None), b"null x, y, partials, coef or dL_dx"),
    (dict(drs=4), b"dL_dx: row stride smaller than the row"),
    (dict(dps=10), b"dL_dx: plane stride smaller than the plane"),
])
def test_backward_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _bwd(lib, **kw) == -1
    assert msg in lib.sgb_last_error()


def test_a_crop_of_a_larger_image_is_a_valid_layout():
    """The plane and row strides of the full image hold the cropped plane: only the sizes and pointers change.
    With no GPU the call then fails in CUDA, not in validation."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_loss_gpu.py")
    lib = _lib.load()
    rc = _fwd(lib, planes=3, h=6, w=5, xps=64, xrs=8, yps=64, yrs=8)
    assert rc == -2
    rc = _fwd(lib, planes=1, h=6, w=5, xps=0, xrs=8, yps=0, yrs=8)   # one plane: its stride is unused
    assert rc == -2


# ---- Python layer

def test_python_layer_rejects_cpu_and_unsupported_arguments():
    from semantic_gaussians_b200.loss_utils import photometric_loss, ssim
    x = torch.rand(3, 16, 16)
    with pytest.raises(ValueError, match="CUDA float32"):
        photometric_loss(x, x.clone())
    with pytest.raises(ValueError, match="CUDA float32"):
        ssim(x, x.clone())
    with pytest.raises(ValueError, match="window_size=11"):
        ssim(x, x.clone(), window_size=7)
    with pytest.raises(ValueError, match="size_average=True"):
        ssim(x, x.clone(), size_average=False)
    with pytest.raises(ValueError, match="must not require grad"):
        photometric_loss(x, x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="must not require grad"):
        ssim(x, x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="at least 100 x 100"):
        photometric_loss(torch.rand(3, 99, 200), torch.rand(3, 99, 200), cut_edge=True)
    with pytest.raises(ValueError, match="at least 100 x 100"):
        photometric_loss(torch.rand(3, 200, 64), torch.rand(3, 200, 64), cut_edge=True)
    with pytest.raises(ValueError, match="shapes differ"):
        photometric_loss(x, torch.rand(3, 16, 17))
    with pytest.raises(ValueError, match=r"\(C,H,W\) or \(N,C,H,W\)"):
        photometric_loss(torch.rand(16, 16), torch.rand(16, 16))
