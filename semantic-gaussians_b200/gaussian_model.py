"""The slice of the reference's GaussianModel that the render / fusion path reads
(model/gaussian_model.py:33-48 activations, :105-144 getters, :188-194 create_semantic).
Density control / optimiser bookkeeping lives in densify.py (mixin), PLY / npz IO in io_formats.py."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def build_rotation(r: torch.Tensor) -> torch.Tensor:
    """utils/general_utils.py:82-104 (normalises the quaternion first)."""
    q = r / torch.sqrt((r * r).sum(dim=1))[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device, dtype=r.dtype)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - w * z)
    R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y)
    R[:, 2, 1] = 2 * (y * z + w * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def build_scaling_rotation(s: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """utils/general_utils.py:106-115: L = R @ diag(s)."""
    L = torch.zeros((s.shape[0], 3, 3), dtype=s.dtype, device=s.device)
    L[:, 0, 0], L[:, 1, 1], L[:, 2, 2] = s[:, 0], s[:, 1], s[:, 2]
    return build_rotation(r) @ L


def strip_symmetric(sym: torch.Tensor) -> torch.Tensor:
    """utils/general_utils.py:66-79: upper triangle (xx, xy, xz, yy, yz, zz)."""
    return torch.stack([sym[:, 0, 0], sym[:, 0, 1], sym[:, 0, 2], sym[:, 1, 1], sym[:, 1, 2], sym[:, 2, 2]], dim=1)


from .densify import DensifyMixin  # noqa: E402


class GaussianModel(DensifyMixin):
    """Parameter container with the reference's raw-parameter conventions: log scales, logit
    opacities, unnormalised quaternions, SH as (P,1,3) dc + (P,15,3) rest."""

    def __init__(self, sh_degree: int = 3):
        # model/gaussian_model.py:47: a fresh model starts at degree 0; train.py:118 raises it with
        # oneupSHdegree() every 1000 iterations (load_ply / load_dynamic_npz / from_activated set the full degree)
        self.active_sh_degree = 0
        self.max_sh_degree = sh_degree
        self._xyz = torch.empty(0)
        self._features_dc = torch.empty(0)
        self._features_rest = torch.empty(0)
        self._scaling = torch.empty(0)
        self._rotation = torch.empty(0)
        self._opacity = torch.empty(0)
        self._features_semantic = torch.empty(0)
        self._times = torch.empty(0)

    @classmethod
    def from_activated(cls, xyz, scales, rotations, opacity, shs=None, sh_degree: int = 3, device="cuda"):
        """Build from activated values (numpy or torch): scales > 0, opacity in (0,1), unit quats."""
        t = lambda a: torch.as_tensor(a, dtype=torch.float32, device=device).contiguous()
        m = cls(sh_degree)
        m.active_sh_degree = sh_degree      # an already-fitted scene (inference / bench): all bands active
        m._xyz = t(xyz)
        m._scaling = torch.log(t(scales))
        m._rotation = t(rotations)
        op = t(opacity).reshape(-1, 1)
        m._opacity = torch.log(op / (1 - op))
        if shs is not None:
            shs = t(shs)
            m._features_dc = shs[:, :1, :].contiguous()
            m._features_rest = shs[:, 1:, :].contiguous()
        return m

    # --- model/gaussian_model.py:105-144
    @property
    def get_scaling(self):
        return torch.exp(self._scaling)

    @property
    def get_rotation(self):
        return F.normalize(self._rotation)

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_features(self):
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    def get_covariance(self, scaling_modifier=1):
        L = build_scaling_rotation(scaling_modifier * self.get_scaling, self._rotation)
        return strip_symmetric(L @ L.transpose(1, 2))

    def get_covariance_rotation(self, scaling_modifier=1, world_rotate=None):
        L = build_scaling_rotation(scaling_modifier * self.get_scaling, self._rotation)
        return strip_symmetric(world_rotate.transpose(0, 1) @ L @ L.transpose(1, 2) @ world_rotate)

    def create_from_pcd(self, points, colors, spatial_lr_scale: float = 1.0, device="cuda"):
        """model/gaussian_model.py:150-186: initialise from a point cloud — SH dc from the colours, isotropic
        log-scales from the mean squared distance to the 3 nearest neighbours (distCUDA2, clamped at 1e-7),
        identity rotations, opacity 0.1.  ``points`` (P,3), ``colors`` (P,3) in [0,1] (numpy or torch)."""
        from .simple_knn._C import distCUDA2
        self.spatial_lr_scale = spatial_lr_scale
        t = lambda a: torch.as_tensor(a).float().to(device)
        xyz = t(points).contiguous()
        fused_color = (t(colors) - 0.5) / 0.28209479177387814                     # RGB2SH, utils/sh_utils.py:118
        n = xyz.shape[0]
        features = torch.zeros((n, 3, (self.max_sh_degree + 1) ** 2), dtype=torch.float32, device=device)
        features[:, :3, 0] = fused_color
        dist2 = torch.clamp_min(distCUDA2(xyz), 0.0000001)
        self._xyz = xyz
        self._features_dc = features[:, :, 0:1].transpose(1, 2).contiguous()
        self._features_rest = features[:, :, 1:].transpose(1, 2).contiguous()
        self._scaling = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
        rots = torch.zeros((n, 4), device=device)
        rots[:, 0] = 1
        self._rotation = rots
        op = 0.1 * torch.ones((n, 1), dtype=torch.float32, device=device)
        self._opacity = torch.log(op / (1 - op))                                   # inverse_sigmoid
        self.max_radii2D = torch.zeros((n,), device=device)
        return self

    def create_semantic(self, dim: int):
        """model/gaussian_model.py:188-194: zero per-Gaussian feature sums and view counts."""
        P, dev = self._xyz.shape[0], self._xyz.device
        self._features_semantic = torch.zeros((P, dim), dtype=torch.float32, device=dev)
        self._times = torch.zeros((P, 1), dtype=torch.float32, device=dev)

    def get_locs_and_features(self, feature_type="all", device=False):
        """model/gaussian_model.py:400-418: the raw xyz (P,3) and the per-Gaussian features the 3D network reads,
        ``"all"``: opacity, SH dc, SH rest, scale, rotation (56 columns at degree 3), ``"color"``: SH dc and rest
        (48).  numpy arrays as the reference returns them, or with ``device=True`` the tensors on the model's
        device with no host copy (voxelize.voxelize_gaussians)."""
        parts = {"all": (self._opacity, self._features_dc, self._features_rest, self._scaling, self._rotation),
                 "color": (self._features_dc, self._features_rest)}
        if feature_type not in parts:
            raise ValueError(f"feature_type must be 'all' or 'color', got {feature_type!r}")
        P = self._xyz.shape[0]
        locs = self._xyz.detach()
        features = torch.cat([t.detach().reshape(P, -1) for t in parts[feature_type]], dim=-1)
        if device:
            return locs, features
        return locs.cpu().numpy().copy(), features.cpu().numpy()

    # --- on-disk formats (model/gaussian_model.py:265-281, :288-344, :346-378) without plyfile
    def save_ply(self, path):
        from .io_formats import save_gaussian_ply
        save_gaussian_ply(path, self)

    def load_ply(self, path, device="cuda"):
        from .io_formats import load_gaussian_ply
        load_gaussian_ply(path, self, device=device)

    def load_dynamic_npz(self, path, t, device="cuda"):
        from .io_formats import load_dynamic_npz
        if not hasattr(self, "_npz_cache"):
            self._npz_cache = {}
        load_dynamic_npz(path, t, self, device=device, cache=self._npz_cache)
