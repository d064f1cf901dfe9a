"""Per-view camera pose correction: learnable offsets for the poses a dataset ships (BundleFusion for ScanNet, SfM for
COLMAP scenes), trained through the rasterizer's camera gradients.

``CameraPoseCorrection(num_cameras, device)`` holds one zero-initialised (N, 6) parameter, row i = (omega, tau) of
camera i, and ``pose(camera, i)`` returns a camera object that ``render*()``, ``fuse_scene`` and ``lift_scene``
accept.  The correction acts in the camera frame,

    p_cam' = R(omega) p_cam + tau,      R(omega) = exp([omega]x)  (axis-angle omega, in radians; tau in scene units)

so W2C' = [[R(omega), tau], [0, 1]] W2C.  In the reference's row-vector convention (``world_view_transform`` = W2C^T):

    world_view_transform' = world_view_transform @ D^T,   D = [[R(omega), tau], [0, 1]]
    full_proj_transform'  = world_view_transform' @ projection_matrix
    camera_center'        = camera_center - world_view_transform[:3, :3] @ (R(omega)^T tau)

(the last is inverse(world_view_transform')[3, :3] in closed form).  Each of the three is computed as the camera's
own tensor plus (f(delta) - f(0)) of one expression f, so at delta = 0 it is bitwise the camera's tensor and the
correction changes nothing until the optimiser moves it.  Every other attribute (image size, FoV, ground truth
image, uid, ...) is read from the wrapped camera.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .scene_synth import get_projection_matrix

# the reference's Camera: getProjectionMatrix(znear=0.01, zfar=100.0, ...)
ZNEAR, ZFAR = 0.01, 100.0


def _hat(w: torch.Tensor) -> torch.Tensor:
    """[w]x, the cross-product matrix of w (3,)."""
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]),
                        torch.stack([-w[1], w[0], z])])


def rotation(omega: torch.Tensor) -> torch.Tensor:
    """R(omega) = I + a [omega]x + b [omega]x^2 with a = sin(t) / t, b = (1 - cos(t)) / t^2, t = |omega| (Rodrigues).
    Below t^2 = 1e-2 a and b are their Taylor series to t^8 (truncation below 1e-17), so the value and the gradient
    are exact and finite at omega = 0; the closed form is evaluated at a safe angle there."""
    t2 = (omega * omega).sum()
    small = t2 < 1e-2
    ts = torch.sqrt(torch.where(small, torch.ones_like(t2), t2))
    a_series = 1 - t2 / 6 * (1 - t2 / 20 * (1 - t2 / 42 * (1 - t2 / 72)))
    b_series = 0.5 * (1 - t2 / 12 * (1 - t2 / 30 * (1 - t2 / 56 * (1 - t2 / 90))))
    a = torch.where(small, a_series, torch.sin(ts) / ts)
    b = torch.where(small, b_series, (1 - torch.cos(ts)) / (ts * ts))
    K = _hat(omega)
    return torch.eye(3, dtype=omega.dtype, device=omega.device) + a * K + b * (K @ K)


def _motion_t(delta: torch.Tensor) -> torch.Tensor:
    """D^T (4, 4) of delta = (omega, tau): the row-vector form of p_cam' = R(omega) p_cam + tau."""
    R = rotation(delta[:3])
    top = torch.cat([R.T, torch.zeros((3, 1), dtype=delta.dtype, device=delta.device)], 1)
    bottom = torch.cat([delta[3:], torch.ones(1, dtype=delta.dtype, device=delta.device)]).reshape(1, 4)
    return torch.cat([top, bottom], 0)


def _moved(wvt: torch.Tensor, proj: torch.Tensor, delta: torch.Tensor):
    """f(delta) of the three tensors: wvt @ D^T, (wvt @ D^T) @ proj and -wvt[:3, :3] @ (R(omega)^T tau)."""
    Dt = _motion_t(delta)
    view = wvt @ Dt
    return view, view @ proj, -(wvt[:3, :3] @ (Dt[:3, :3] @ delta[3:]))


def _anchored(orig: torch.Tensor, f0: torch.Tensor, f: torch.Tensor) -> torch.Tensor:
    """orig + f(delta) - f(0), written so that it is bitwise orig at delta = 0: f(0) - f(delta) is then +0, and
    x - (+0) is x for every x (a signed zero included)."""
    return orig - (f0 - f)


class CorrectedCamera:
    """A camera whose world_view_transform, full_proj_transform and camera_center are those of ``camera`` moved by the
    correction ``delta`` (differentiable functions of it); every other attribute is ``camera``'s."""

    def __init__(self, camera, delta: torch.Tensor):
        wvt = camera.world_view_transform
        proj = getattr(camera, "projection_matrix", None)
        if proj is None:
            proj = torch.as_tensor(get_projection_matrix(ZNEAR, ZFAR, camera.FoVx, camera.FoVy).T.copy(),
                                   device=wvt.device)
        proj = torch.as_tensor(proj, dtype=wvt.dtype, device=wvt.device)
        delta = delta.to(wvt.dtype)
        self._camera = camera
        self.projection_matrix = proj
        with torch.no_grad():   # f(0) by the same expressions as f(delta), so the two agree bitwise at delta = 0
            f0 = _moved(wvt, proj, torch.zeros_like(delta))
        f = _moved(wvt, proj, delta)
        full = torch.as_tensor(camera.full_proj_transform, device=wvt.device)
        center = torch.as_tensor(camera.camera_center, device=wvt.device)
        self.world_view_transform, self.full_proj_transform, self.camera_center = (
            _anchored(o, a, b) for o, a, b in zip((wvt, full, center), f0, f))

    def __getattr__(self, name):  # only reached for attributes not set in __init__
        return getattr(self.__dict__["_camera"], name)


class CameraPoseCorrection(nn.Module):
    """One learnable pose correction per training camera: ``delta`` (num_cameras, 6), rows (omega, tau), zeros at
    start.  ``self(camera, index)`` is ``camera`` moved by row ``index`` (module docstring).  Optimise it with its own
    optimiser (for example ``torch.optim.Adam(pose.parameters(), lr=1e-4)``); the rasterizer's backward fills the
    camera gradients whenever the camera tensors require grad."""

    def __init__(self, num_cameras: int, device=None):
        super().__init__()
        self.delta = nn.Parameter(torch.zeros((int(num_cameras), 6), device=device))

    def forward(self, camera, index: int) -> CorrectedCamera:
        return CorrectedCamera(camera, self.delta[index])
