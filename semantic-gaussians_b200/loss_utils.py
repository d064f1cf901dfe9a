"""RGB training loss on the GPU: the L1 + D-SSIM loss of the reference's training step (train.py:141-149) and
the ``ssim`` of utils/loss_utils.py:38-72, each as one fused forward kernel and one fused backward kernel
(csrc/loss.cu) instead of five depthwise convolutions, ~15 full-size temporaries and their autograd replay.

``photometric_loss(image, gt, lambda_dssim=0.2, cut_edge=False) -> (loss, l1)``
        loss = (1 - lambda_dssim) * L1(image, gt) + lambda_dssim * (1 - ssim(image, gt)),  on the border-cropped
        images when ``cut_edge`` (``image[:, h//100 : -(h//100), w//100 : -(w//100)]``, as train.py does).
``ssim(img1, img2, window_size=11, size_average=True)``
        mean SSIM of (C,H,W) or (N,C,H,W) images, a drop-in for utils/loss_utils.py:ssim.

Gradient flows to the first (rendered) image only.  Neither call synchronises the host."""
from __future__ import annotations

from typing import Tuple

import torch

from . import _lib


def _check(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
        raise ValueError(f"{name} must be a CUDA float32 tensor (the fused loss has no CPU path)")
    return t


def _plane_layout(t: torch.Tensor):
    """(planes, plane stride, row stride) of a (C,H,W) / (N,C,H,W) view whose planes share one stride and whose
    pixel stride is 1, or None when the layout cannot be addressed that way."""
    h, w = t.shape[-2:]
    if t.stride(-1) != 1 and w > 1:
        return None
    rs = t.stride(-2) if h > 1 else w
    if t.ndim == 3:
        planes, ps = t.shape[0], t.stride(0)
    else:
        n, c = t.shape[:2]
        planes = n * c
        if c == 1:
            ps = t.stride(0)
        elif n == 1 or t.stride(0) == c * t.stride(1):
            ps = t.stride(1)
        else:
            return None
    if planes == 1:
        ps = h * rs
    if rs < w or ps < (h - 1) * rs + w:
        return None          # overlapping rows or planes (expanded views): make a contiguous copy
    return planes, ps, rs


def _addressable(t: torch.Tensor) -> torch.Tensor:
    """t itself when its planes can be passed to the kernels as (pointer, plane stride, row stride), else a copy."""
    return t if _plane_layout(t) is not None else t.contiguous()


def _crop(t: torch.Tensor, cut_edge: bool) -> torch.Tensor:
    if not cut_edge:
        return t
    h, w = t.shape[-2:]
    ch, cw = h // 100, w // 100
    return t[..., ch:h - ch, cw:w - cw]


def _args(t: torch.Tensor):
    planes, ps, rs = _plane_layout(t)
    return t.data_ptr(), ps, rs


class _FusedLoss(torch.autograd.Function):
    """value = k0 + k1 * mean|x - y| + k2 * mean SSIM(x, y) over the (cropped) planes.  One native call each way."""

    @staticmethod
    def forward(ctx, x, y, cut_edge: bool, k0: float, k1: float, k2: float):
        xc, yc = _crop(x, cut_edge), _crop(y, cut_edge)
        planes, _, _ = _plane_layout(xc)
        h, w = xc.shape[-2:]
        n = xc.numel()
        want_grad = ctx.needs_input_grad[0]
        sums = torch.empty(2, dtype=torch.float64, device=x.device)
        partials = torch.empty((3, planes, h, w), dtype=torch.float32, device=x.device) if want_grad else None
        with torch.cuda.device(x.device):
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _lib.check(_lib.load().sgb_photometric_forward(
                planes, h, w, *_args(xc), *_args(yc), sums.data_ptr(),
                partials.data_ptr() if partials is not None else None, stream), "sgb_photometric_forward")
        means = sums / n                                   # [L1, mean SSIM], float64 on the device
        value = (k0 + k1 * means[0] + k2 * means[1]).float()
        l1 = means[0].float()
        ctx.mark_non_differentiable(l1)
        if want_grad:
            ctx.save_for_backward(x, y, partials)
        ctx.cfg = (cut_edge, k1 / n, k2 / n)
        return value, l1

    @staticmethod
    def backward(ctx, grad_value, grad_l1):
        x, y, partials = ctx.saved_tensors
        cut_edge, c1, c2 = ctx.cfg
        g = grad_value.reshape(1).float()
        coef = torch.cat((g * c1, g * c2)).contiguous()    # stays on the device: backward never syncs the host
        dx = (torch.zeros if cut_edge else torch.empty)(x.shape, dtype=torch.float32, device=x.device)
        xc, yc, dxc = _crop(x, cut_edge), _crop(y, cut_edge), _crop(dx, cut_edge)
        planes, _, _ = _plane_layout(xc)
        h, w = xc.shape[-2:]
        with torch.cuda.device(x.device):
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _lib.check(_lib.load().sgb_photometric_backward(
                planes, h, w, *_args(xc), *_args(yc), partials.data_ptr(), coef.data_ptr(), *_args(dxc), stream),
                "sgb_photometric_backward")
        return dx, None, None, None, None, None


def _prepare(img: torch.Tensor, target: torch.Tensor, cut_edge: bool):
    # shape and autograd checks first, then the device: each mistake is reported as itself
    for t, name in ((img, "image"), (target, "target")):
        if not isinstance(t, torch.Tensor) or t.ndim not in (3, 4):
            raise ValueError(f"{name} must be a (C,H,W) or (N,C,H,W) tensor")
    if target.requires_grad:
        raise ValueError("the target image must not require grad: the fused loss differentiates the rendered "
                         "image only (detach the target)")
    if img.shape != target.shape:
        raise ValueError(f"image and target shapes differ: {tuple(img.shape)} vs {tuple(target.shape)}")
    if cut_edge and (img.shape[-2] < 100 or img.shape[-1] < 100):
        raise ValueError(f"cut_edge needs an image of at least 100 x 100 pixels (got {img.shape[-2]} x "
                         f"{img.shape[-1]}): below that the border crop h//100 : -(h//100) is empty")
    if img.numel() == 0:
        raise ValueError("empty image")
    x, y = _check(img, "image"), _check(target, "target")
    if x.device != y.device:
        raise ValueError("image and target are on different devices")
    return _addressable(x), _addressable(y)


def photometric_loss(image: torch.Tensor, gt: torch.Tensor, lambda_dssim: float = 0.2,
                     cut_edge: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """train.py:141-149 in one fused forward and one fused backward:

        l1   = |image - gt|.mean()
        loss = (1 - lambda_dssim) * l1 + lambda_dssim * (1 - ssim(image, gt))

    over ``image[..., h//100 : h - h//100, w//100 : w - w//100]`` when ``cut_edge`` (the crop is taken through
    strides; the gradient is zero outside it).  image / gt: CUDA float32 (C,H,W) or (N,C,H,W).
    Returns (loss: differentiable 0-d float32, l1: detached 0-d float32), both on the device."""
    x, y = _prepare(image, gt, cut_edge)
    lam = float(lambda_dssim)
    return _FusedLoss.apply(x, y, bool(cut_edge), lam, 1.0 - lam, -lam)


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True) -> torch.Tensor:
    """Mean SSIM of img1 against img2 (utils/loss_utils.py:ssim): (C,H,W) or (N,C,H,W) CUDA float32, 11x11
    Gaussian window (sigma 1.5) over zero padding.  Differentiable in img1 only."""
    if window_size != 11:
        raise ValueError("ssim: only window_size=11 is implemented (the reference's only use)")
    if not size_average:
        raise ValueError("ssim: only size_average=True is implemented (the reference's only use)")
    x, y = _prepare(img1, img2, False)
    return _FusedLoss.apply(x, y, False, 0.0, 0.0, 1.0)[0]
