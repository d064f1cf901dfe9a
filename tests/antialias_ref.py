"""Float64 restatement of the anti-aliasing filter (semantic-gaussians_b200/csrc/geom_grad.cuh aa_scale /
aa_cov_grad, preprocess_kernel<true>, geom_backward_kernel<*, true>), for tests/test_antialias_*.py.

With C0 = (a0, b; b, c0) the screen covariance before the 0.3 px^2 dilation and C = C0 + 0.3 I:
    r = det C0 / det C,   h = sqrt(max(eps, r)),   o_eff = o h,   eps = 2.5e-5
and, with g = dL/do_eff: dL/do = h g, and for r > eps dL/dC0 gains (o g / (2 h)) dr/dC0 (0 on the floor branch).
The screen covariance is restated from (means3D, cov3D) and the camera the way the forward forms it (frustum-clamped
Jacobian), in float64 torch so that autograd gives the chain to means3D, cov3D, scales and rotations."""
import math

import numpy as np
import torch

S = 0.3
EPS = 2.5e-5


def h_of(a0, b, c0):
    """(r, h, active) of float64 arrays a0, b, c0."""
    a0, b, c0 = (np.asarray(x, np.float64) for x in (a0, b, c0))
    r = (a0 * c0 - b * b) / ((a0 + S) * (c0 + S) - b * b)
    return r, np.sqrt(np.maximum(EPS, r)), r > EPS


def dr_dcov(a0, b, c0):
    """dr/d(a0, b, c0), b the off-diagonal value, (n, 3) float64."""
    a0, b, c0 = (np.asarray(x, np.float64) for x in (a0, b, c0))
    D2 = ((a0 + S) * (c0 + S) - b * b) ** 2
    return np.stack([S * (c0 * c0 + S * c0 + b * b) / D2, -2 * S * b * (a0 + c0 + S) / D2,
                     S * (a0 * a0 + S * a0 + b * b) / D2], -1)


def cov6_from_factors(scales, rotations, mod=1.0):
    """World covariance (n, 6) of R diag(mod s)^2 R^T, the quaternion (r, x, y, z) used as given."""
    r, x, y, z = rotations.unbind(-1)
    R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                     torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                     torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], -2)
    L = R * (mod * scales)[:, None, :]
    Sg = L @ L.transpose(1, 2)
    return torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], -1)


def screen_cov0(means3D, cov6, view, W, H, tan_fovx, tan_fovy):
    """(a0, b, c0) of every Gaussian, float64 torch (differentiable in means3D and cov6).  view: the 16 floats of the
    viewmatrix as the rasterizer takes them (element (row i, col j) at [4 j + i])."""
    v = torch.as_tensor(np.asarray(view, np.float64).reshape(-1), device=means3D.device)
    Wm = torch.stack([torch.stack([v[4 * j + i] for j in range(3)]) for i in range(3)])
    t = means3D @ Wm.T + v[12:15]
    fx, fy = W / (2.0 * tan_fovx), H / (2.0 * tan_fovy)
    lx, ly = 1.3 * tan_fovx, 1.3 * tan_fovy
    tz = t[:, 2]
    # t.x = clamp(t.x / t.z) t.z; where the clamp bites, the reference's backward holds that clamped t.x fixed
    # (backward.cu:252-253 mask only the direct terms), and so does this restatement
    ux, uy = t[:, 0] / tz, t[:, 1] / tz
    tx = torch.where(ux.abs() > lx, (torch.clamp(ux, -lx, lx) * tz).detach(), t[:, 0])
    ty = torch.where(uy.abs() > ly, (torch.clamp(uy, -ly, ly) * tz).detach(), t[:, 1])
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * tx / (tz * tz)], -1),
                     torch.stack([zero, fy / tz, -fy * ty / (tz * tz)], -1)], -2)
    A = J @ Wm
    c = cov6
    Sg = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], -1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], -1),
                      torch.stack([c[:, 2], c[:, 4], c[:, 5]], -1)], -2)
    C0 = A @ Sg @ A.transpose(1, 2)
    return C0[:, 0, 0], C0[:, 0, 1], C0[:, 1, 1]


def r_torch(a0, b, c0):
    return (a0 * c0 - b * b) / ((a0 + S) * (c0 + S) - b * b)


def footprint(opacity, a0, b, c0):
    """o 2 pi sqrt(det C0): the integral of an undilated Gaussian of opacity o over the image plane, in pixels."""
    return np.asarray(opacity, np.float64) * 2 * math.pi * np.sqrt(np.asarray(a0) * c0 - np.asarray(b) ** 2)
