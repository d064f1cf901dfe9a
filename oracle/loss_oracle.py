"""TEST INFRASTRUCTURE ONLY — numpy float64 statement of the photometric training loss and of its analytic
gradient, the checker for semantic-gaussians_b200/csrc/loss.cu (never imported by the product path).

The loss is train.py:141-149:  (1 - lam) * mean|x - y| + lam * (1 - mean SSIM(x, y)),  optionally on the images
with a border of h//100 rows and w//100 columns removed.  SSIM is computed per plane (one channel of one image)
with the 11-tap Gaussian window (sigma 1.5) applied along rows and then columns, over zero padding.
tests/test_loss_cpu.py pins both the value and the gradient against torch float64 autograd of the reference's
torch expressions."""
import math

import numpy as np

C1 = 0.01 ** 2
C2 = 0.03 ** 2
RADIUS = 5


def window_taps() -> np.ndarray:
    """The 11 taps as the reference makes them: exp values rounded to fp32, divided by their fp32 sum (torch's
    sum of these 11 values is the correctly rounded one, which a float64 sum rounded to fp32 reproduces)."""
    g = np.array([math.exp(-((i - RADIUS) ** 2) / (2 * 1.5 ** 2)) for i in range(2 * RADIUS + 1)], np.float32)
    return (g / np.float32(g.astype(np.float64).sum())).astype(np.float32)


def blur(a: np.ndarray, taps: np.ndarray = None) -> np.ndarray:
    """Zero-padded 11 x 11 window over the last two axes of a, as one pass along columns and one along rows."""
    t = (window_taps() if taps is None else taps).astype(np.float64)
    a = np.asarray(a, np.float64)
    h, w = a.shape[-2:]
    pad = [(0, 0)] * (a.ndim - 2) + [(RADIUS, RADIUS), (RADIUS, RADIUS)]
    p = np.pad(a, pad)
    rows = sum(t[k] * p[..., :, k:k + w] for k in range(len(t)))          # (.., h + 10, w)
    return sum(t[k] * rows[..., k:k + h, :] for k in range(len(t)))       # (.., h, w)


def crop_slices(h: int, w: int, cut_edge: bool):
    if not cut_edge:
        return slice(0, h), slice(0, w)
    ch, cw = h // 100, w // 100
    if ch == 0 or cw == 0:
        raise ValueError("cut_edge needs an image of at least 100 x 100 pixels")
    return slice(ch, h - ch), slice(cw, w - cw)


def ssim_terms(x: np.ndarray, y: np.ndarray):
    """Per-pixel SSIM map S and the three maps (a, b, c) with
    d(sum S)/dx = blur(a) + 2 x blur(b) + y blur(c)."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    mx, my = blur(x), blur(y)
    vx = blur(x * x) - mx * mx
    vy = blur(y * y) - my * my
    cxy = blur(x * y) - mx * my
    a1, a2 = 2 * mx * my + C1, 2 * cxy + C2
    b1, b2 = mx * mx + my * my + C1, vx + vy + C2
    s = a1 * a2 / (b1 * b2)
    # partial derivatives of S with respect to the window means and second moments
    da = 2 * my * a2 / (b1 * b2) - 2 * mx * s / b1 + 2 * mx * s / b2 - my * 2 * a1 / (b1 * b2)
    db = -s / b2
    dc = 2 * a1 / (b1 * b2)
    return s, da, db, dc


def ssim_grad_sum(x: np.ndarray, y: np.ndarray):
    """(sum of the SSIM map, d(sum)/dx) over every plane of x (shape (..., h, w))."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    s, da, db, dc = ssim_terms(x, y)
    return s.sum(), blur(da) + 2 * x * blur(db) + y * blur(dc)


def ssim(x: np.ndarray, y: np.ndarray):
    """(mean SSIM, its gradient with respect to x)."""
    total, g = ssim_grad_sum(x, y)
    n = np.asarray(x).size
    return total / n, g / n


def photometric_loss(x: np.ndarray, y: np.ndarray, lam: float = 0.2, cut_edge: bool = False):
    """(loss, l1, d loss / dx) for (C,H,W) or (N,C,H,W) images; the gradient is full-size, zero outside the crop."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    rs, cs = crop_slices(x.shape[-2], x.shape[-1], cut_edge)
    xc, yc = x[..., rs, cs], y[..., rs, cs]
    n = xc.size
    l1 = np.abs(xc - yc).sum() / n
    ssum, sgrad = ssim_grad_sum(xc, yc)
    loss = (1 - lam) * l1 + lam * (1 - ssum / n)
    grad = np.zeros_like(x)
    grad[..., rs, cs] = (1 - lam) / n * np.sign(xc - yc) - lam / n * sgrad
    return loss, l1, grad
