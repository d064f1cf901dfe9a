"""Synthetic scenes and cameras for tests, golden fixtures and bench (numpy only, except the torch voxel cloud of
``surface_voxels``).

The reference ships no generator; its distributions are the blob and room scenes below.  Camera matrices
follow the reference's conventions exactly:

* ``world_view_transform`` = W2C transposed            (scene/camera.py:87)
* ``projection_matrix``    = getProjectionMatrix(...)ᵀ  (utils/graphics_utils.py:56-76)
* ``full_proj_transform``  = world_view @ projection   (scene/camera.py:91-93)
* ``camera_center``        = inverse(world_view)[3,:3] (scene/camera.py:94)

Everything is deterministic in ``seed`` (numpy Generator PCG64), so fixtures only need to
store outputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

ZNEAR, ZFAR = 0.01, 100.0  # scene/camera.py:81-82


def get_world2view2(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """W2C 4x4 float32; R is camera-to-world rotation, t the W2C translation
    (utils/graphics_utils.py:42-53 with translate=0, scale=1)."""
    Rt = np.zeros((4, 4), dtype=np.float64)
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    C2W = np.linalg.inv(Rt)
    Rt = np.linalg.inv(C2W)
    return np.float32(Rt)


def get_projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> np.ndarray:
    """utils/graphics_utils.py:56-76 (float32 like the torch.zeros(4,4) it fills)."""
    tan_y = math.tan(fovy / 2)
    tan_x = math.tan(fovx / 2)
    top, right = tan_y * znear, tan_x * znear
    bottom, left = -top, -right
    P = np.zeros((4, 4), dtype=np.float32)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


@dataclass
class SynthCamera:
    """Duck-type of the reference's ``Camera`` / ``MiniCam`` fields that render() reads."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: np.ndarray   # (4,4) f32, W2C^T
    projection_matrix: np.ndarray      # (4,4) f32, P^T
    full_proj_transform: np.ndarray    # (4,4) f32, (P W2C)^T
    camera_center: np.ndarray          # (3,) f32
    znear: float = ZNEAR
    zfar: float = ZFAR

    @property
    def tanfovx(self) -> float:
        return math.tan(self.FoVx * 0.5)

    @property
    def tanfovy(self) -> float:
        return math.tan(self.FoVy * 0.5)

    def intrinsics(self) -> np.ndarray:
        """4x4 pinhole intrinsics in pixels (for fusion's PointCloudToImageMapper)."""
        fx = self.image_width / (2 * self.tanfovx)
        fy = self.image_height / (2 * self.tanfovy)
        K = np.eye(4)
        K[0, 0], K[1, 1] = fx, fy
        K[0, 2], K[1, 2] = self.image_width / 2, self.image_height / 2
        return K


def look_at_camera(eye, target, width: int, height: int, fovx_deg: float = 60.0,
                   up=(0.0, 0.0, 1.0)) -> SynthCamera:
    """Camera at ``eye`` looking at ``target`` (+z forward, +x right, +y down, COLMAP-like)."""
    eye = np.asarray(eye, np.float64)
    target = np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    upv = np.asarray(up, np.float64)
    x = np.cross(z, upv)
    if np.linalg.norm(x) < 1e-8:
        x = np.cross(z, np.array([0.0, 1.0, 0.0]))
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    Rw2c = np.stack([x, y, z], axis=0)
    R = Rw2c.T                       # camera-to-world, as Camera(R=...) stores it
    t = -Rw2c @ eye
    fovx = math.radians(fovx_deg)
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * height / width)
    w2c = get_world2view2(R, t)
    wvt = np.ascontiguousarray(w2c.T)
    proj = np.ascontiguousarray(get_projection_matrix(ZNEAR, ZFAR, fovx, fovy).T)
    full = (wvt @ proj).astype(np.float32)
    center = np.linalg.inv(wvt)[3, :3].astype(np.float32)
    return SynthCamera(width, height, fovx, fovy, wvt, proj, np.ascontiguousarray(full),
                       np.ascontiguousarray(center))


def orbit_cameras(n_views: int, width: int, height: int, radius: float = 3.0,
                  height_z: float = 0.4, fovx_deg: float = 60.0, target=(0, 0, 0)):
    cams = []
    for i in range(n_views):
        a = 2 * math.pi * i / max(n_views, 1) + 0.1
        eye = (radius * math.cos(a), radius * math.sin(a), height_z)
        cams.append(look_at_camera(eye, target, width, height, fovx_deg))
    return cams


def room_cameras(n_views: int, width: int, height: int, fovx_deg: float = 60.0):
    """Cameras inside the 'room' scene at height 0, on a small circle, looking outward-ish."""
    cams = []
    for i in range(n_views):
        a = 2 * math.pi * i / max(n_views, 1) + 0.05
        eye = (1.5 * math.cos(a), 1.5 * math.sin(a), 0.0)
        tgt = (-2.5 * math.cos(a + 0.3), -2.5 * math.sin(a + 0.3), 0.0)
        cams.append(look_at_camera(eye, tgt, width, height, fovx_deg))
    return cams


@dataclass
class SynthScene:
    xyz: np.ndarray        # (P,3) f32
    scales: np.ndarray     # (P,3) f32  (already exp-activated, >0)
    rotations: np.ndarray  # (P,4) f32  unit quaternions (w,x,y,z)
    opacity: np.ndarray    # (P,1) f32  in (0,1)
    shs: Optional[np.ndarray] = None       # (P,16,3) f32
    features: Optional[np.ndarray] = None  # (P,C) f32

    @property
    def P(self) -> int:
        return self.xyz.shape[0]


def make_scene(P: int, seed: int = 0, kind: str = "blob", sh: bool = False, channels: int = 0,
               scale_mean: float = 0.02) -> SynthScene:
    """blob U([-1.3,1.3]^3) (model/gaussian_model.py:158) or room
    U([-4,4]x[-4,4]x[-1.5,1.5]); log-normal scales; random unit quaternions; sigmoid(N(0,2^2))
    opacity; SH dc U(-1.5,1.5) rest N(0,0.1^2); L2-normalised N(0,1) feature rows."""
    rng = np.random.default_rng(seed)
    if kind == "blob":
        xyz = rng.uniform(-1.3, 1.3, size=(P, 3))
    elif kind == "room":
        xyz = np.stack([rng.uniform(-4, 4, P), rng.uniform(-4, 4, P), rng.uniform(-1.5, 1.5, P)], 1)
    else:
        raise ValueError(kind)
    log_s = rng.normal(math.log(scale_mean), 0.5, size=(P, 3))
    log_s = np.clip(log_s, math.log(0.002), math.log(0.3))
    scales = np.exp(log_s)
    q = rng.normal(size=(P, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    opacity = 1.0 / (1.0 + np.exp(-rng.normal(0.0, 2.0, size=(P, 1))))
    shs = None
    if sh:
        shs = np.concatenate([rng.uniform(-1.5, 1.5, size=(P, 1, 3)),
                              rng.normal(0, 0.1, size=(P, 15, 3))], axis=1).astype(np.float32)
    feats = None
    if channels > 0:
        # generate in float32 chunks to bound memory at 1M x 256+
        feats = np.empty((P, channels), dtype=np.float32)
        step = 1 << 16
        for s in range(0, P, step):
            f = rng.standard_normal(size=(min(step, P - s), channels), dtype=np.float32)
            f /= np.linalg.norm(f, axis=1, keepdims=True)
            feats[s:s + f.shape[0]] = f
    return SynthScene(xyz.astype(np.float32), scales.astype(np.float32), q.astype(np.float32),
                      opacity.astype(np.float32), shs, feats)


def surface_points(n: int, seed: int = 0) -> np.ndarray:
    """(n,3) float32 points on the floor (z = -1.5) and the four walls (x, y = +-4) of the `room` scene, by area, with
    1 cm jitter: stand-ins for the scan vertices a per-point 3D evaluation labels."""
    rng = np.random.default_rng(seed)
    areas = np.array([64.0, 24.0, 24.0, 24.0, 24.0])
    which = rng.choice(5, size=n, p=areas / areas.sum())
    p = np.stack([rng.uniform(-4, 4, n), rng.uniform(-4, 4, n), rng.uniform(-1.5, 1.5, n)], 1)
    p[which == 0, 2] = -1.5
    for i, (axis, val) in enumerate(((0, -4.0), (0, 4.0), (1, -4.0), (1, 4.0))):
        p[which == i + 1, axis] = val
    return (p + rng.normal(0.0, 0.01, (n, 3))).astype(np.float32)


def surface_voxels(P: int, dev, seed: int = 0):
    """Voxel rows and features of P points on the floor (z = -1.5) and the four walls (x, y = +-4) of the 8 x 8 x 3 m
    room, by area, with 1 cm jitter, at voxel size 0.02: closer to the occupancy of a scanned scene than the
    volumetric `room` Gaussians.  Returns int32 rows (1, x, y, z) and 56 N(0, 1) features per voxel, on ``dev``."""
    import torch

    from .voxelize import voxel_indices
    g = torch.Generator(device=dev).manual_seed(seed)
    u = lambda n, lo, hi: torch.rand(n, device=dev, generator=g) * (hi - lo) + lo   # noqa: E731
    areas = torch.tensor([64.0, 24.0, 24.0, 24.0, 24.0])
    counts = (areas / areas.sum() * P).long().tolist()
    parts = [torch.stack([u(counts[0], -4, 4), u(counts[0], -4, 4), torch.full((counts[0],), -1.5, device=dev)], 1)]
    for i, (axis, val) in enumerate(((0, -4.0), (0, 4.0), (1, -4.0), (1, 4.0))):
        n = counts[1 + i]
        p = torch.stack([u(n, -4, 4), u(n, -4, 4), u(n, -1.5, 1.5)], 1)
        p[:, axis] = val
        parts.append(p)
    xyz = torch.cat(parts) + torch.randn(sum(counts), 3, device=dev, generator=g) * 0.01
    T = [[50.0, 0, 0, 0], [0, 50.0, 0, 0], [0, 0, 50.0, 0]]
    _, _, vox = voxel_indices(xyz.float().contiguous(), T)
    locs = torch.cat([torch.ones((vox.shape[0], 1), dtype=torch.int32, device=dev), vox], 1)
    feats = torch.randn(vox.shape[0], 56, device=dev, generator=g)
    return locs, feats
