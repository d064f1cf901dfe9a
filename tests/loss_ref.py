"""The reference's photometric loss as plain torch expressions (utils/loss_utils.py:18-72, train.py:141-149),
restated for the tests: autograd of these is what the fused loss and the numpy oracle are checked against."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def taps_fp32() -> torch.Tensor:
    """gaussian(11, 1.5): fp32 exp values divided by their fp32 sum (loss_utils.py:26-28)."""
    g = torch.tensor([math.exp(-((i - 5) ** 2) / float(2 * 1.5 ** 2)) for i in range(11)], dtype=torch.float32)
    return g / g.sum()


def window(dtype=torch.float32, device="cpu", separable_fp64=False) -> torch.Tensor:
    """The 11x11 window.  Default: as the reference builds it (fp32 outer product, then cast).  With
    ``separable_fp64`` the outer product of the same fp32 taps is taken in float64: exactly what two separable
    11-tap passes apply, so an fp64 computation over it has no window rounding at all."""
    g = taps_fp32()
    if separable_fp64:
        w2 = torch.outer(g.double(), g.double())
    else:
        w2 = g[:, None].mm(g[None, :])
    return w2.to(dtype=dtype, device=device)


def ssim_torch(img1: torch.Tensor, img2: torch.Tensor, win2d: torch.Tensor) -> torch.Tensor:
    """loss_utils.py:_ssim with size_average=True, for (C,H,W) or (N,C,H,W)."""
    ch = img1.size(-3)
    w = win2d.to(img1.dtype).expand(ch, 1, 11, 11).contiguous()
    mu1 = F.conv2d(img1, w, padding=5, groups=ch)
    mu2 = F.conv2d(img2, w, padding=5, groups=ch)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = F.conv2d(img1 * img1, w, padding=5, groups=ch) - mu1_sq
    sigma2_sq = F.conv2d(img2 * img2, w, padding=5, groups=ch) - mu2_sq
    sigma12 = F.conv2d(img1 * img2, w, padding=5, groups=ch) - mu1_mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    return ssim_map.mean()


def crop(t: torch.Tensor, cut_edge: bool) -> torch.Tensor:
    if not cut_edge:
        return t
    h, w = t.shape[-2:]
    ch, cw = h // 100, w // 100
    return t[..., ch:-ch, cw:-cw]


def photometric_torch(image: torch.Tensor, gt: torch.Tensor, win2d: torch.Tensor, lam: float = 0.2,
                      cut_edge: bool = False):
    """train.py:141-149: (loss, l1)."""
    x, y = crop(image, cut_edge), crop(gt, cut_edge)
    l1 = torch.abs(x - y).mean()
    return (1.0 - lam) * l1 + lam * (1.0 - ssim_torch(x, y, win2d)), l1
