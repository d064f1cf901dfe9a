"""The 3D distillation sample of dataset/feature_dataset.py and dataset/augmentation.py on the GPU.

``FeatureDataset[i]`` reads one scene's Gaussian PLY and fused-feature file and returns what the reference's
``__getitem__`` returns, as CUDA tensors and bitwise equal to the reference's after ``.cuda()``.  With ``aug=True``
the steps run in the reference's order: ``ElasticDistortion`` (two passes), ``Voxelizer.voxelize`` with a random
rotation and scale (``voxelize.Voxelizer``), the target rows (``voxelize.distill_targets``), then the random flip of
x and y.  Every random number is drawn on the host from ``random`` and ``np.random`` in the reference's order, so
``random.seed(s); np.random.seed(s)`` gives the reference's sample.

Host reads per sample: the 6 per-axis bounds of each distortion pass (they fix the noise grid, and so how many
normals are drawn) and the voxel count.  The noise grids are small ((42, 42, 17, 3) and (13, 13, 7, 3) for an
8 x 8 x 3 m room) and are drawn and smoothed on the host with numpy / scipy, then uploaded; the per-point lookup runs
in ``sgb_elastic_displace``.

Numerics are pinned to numpy 2 and scipy 1.18: the grid size is ``(max - min) // granularity`` in the input's dtype
(float32 floor division on the first pass, under numpy 2's promotion rules), the axes are ``np.linspace`` of the
reference's bounds, and the lookup restates scipy 1.18's ``RegularGridInterpolator`` (see csrc/elastic.cu).  A
numpy with other promotion rules can change the grid size, and then every later draw.

The dataset returns CUDA tensors, so a ``DataLoader`` over it runs with ``num_workers=0``."""
from __future__ import annotations

import ctypes as C
import os
import random

import numpy as np
import scipy.ndimage
import torch

from . import _lib
from .gaussian_model import GaussianModel
from .io_formats import load_gaussian_ply
from .voxelize import Voxelizer, distill_targets

# dataset/augmentation.py:170-172: one 3-tap box filter per axis
_BLUR = [np.ones(shape).astype("float32") / 3 for shape in ((3, 1, 1, 1), (1, 3, 1, 1), (1, 1, 3, 1))]


def _to_cuda(coords):
    if isinstance(coords, torch.Tensor):
        if not coords.is_cuda:
            raise ValueError("coords must be a numpy array or a CUDA tensor")
        return coords
    return torch.from_numpy(np.ascontiguousarray(coords)).cuda()


def noise_grid(coords_min: np.ndarray, coords_max: np.ndarray, granularity: float):
    """The host half of dataset/augmentation.py ``elastic_distortion``: from the per-axis min and max of the cloud (two
    (3,) arrays in the cloud's dtype), draw the (nx, ny, nz, 3) fp32 noise from ``np.random``, smooth it twice with
    the three box filters and return it with the three ``np.linspace`` axes.  numpy / scipy make the same calls as
    the reference, so the result is the reference's by construction."""
    # (coords - coords_min).max(0) is max - min: rounding is monotonic
    noise_dim = ((coords_max - coords_min) // granularity).astype(int) + 3
    noise = np.random.randn(*noise_dim, 3).astype(np.float32)
    for _ in range(2):
        for blur in _BLUR:
            noise = scipy.ndimage.convolve(noise, blur, mode="constant", cval=0)
    ax = [np.linspace(d_min, d_max, d)
          for d_min, d_max, d in zip(coords_min - granularity, coords_min + granularity * (noise_dim - 2), noise_dim)]
    if not all((np.diff(a) > 0).all() for a in ax):
        raise ValueError("the noise grid's axes are not strictly ascending (coordinates too large for the granularity)")
    return noise, ax


class ElasticDistortion:
    """dataset/augmentation.py ``ElasticDistortion``: with probability 0.95 (``random.random() < 0.95``), one
    distortion pass per (granularity, magnitude) of ``distortion_params``, each drawing
    ``np.random.randn(*noise_dim, 3)``.  A (P, 3) numpy array gives a float64 numpy array, a CUDA float32 / float64
    tensor a CUDA float64 tensor.  When the gate skips, the input itself is returned, as the reference returns it."""

    def __init__(self, distortion_params):
        self.distortion_params = distortion_params

    def elastic_distortion(self, coords, granularity, magnitude):
        """One pass on a numpy array or CUDA tensor (P, 3), float32 or float64."""
        xyz = _to_cuda(coords)
        if xyz.dtype not in (torch.float32, torch.float64) or xyz.ndim != 2 or xyz.shape[1] != 3 or not len(xyz):
            raise ValueError(f"coords must be (P, 3) float32 or float64 with P > 0, got {tuple(xyz.shape)} "
                             f"{xyz.dtype}")
        xyz = xyz.contiguous()
        # one read of 6 values, in xyz's dtype
        bounds = torch.cat([xyz.amin(0), xyz.amax(0)]).cpu().numpy()
        if not np.isfinite(bounds).all():
            raise ValueError("coords has a non-finite coordinate")
        noise, ax = noise_grid(bounds[:3], bounds[3:], granularity)
        dev = xyz.device
        grid = torch.from_numpy(np.ascontiguousarray(noise, np.float32)).to(dev)
        axes = torch.from_numpy(np.concatenate(ax).astype(np.float64)).to(dev)
        out = torch.empty(xyz.shape, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(_lib.load().sgb_elastic_displace(len(xyz), xyz.data_ptr(), int(xyz.dtype == torch.float64),
                                                        grid.data_ptr(), *noise.shape[:3],
                                                        axes.data_ptr(), C.c_double(magnitude), out.data_ptr(),
                                                        stream), "sgb_elastic_displace")
        return out if isinstance(coords, torch.Tensor) else out.cpu().numpy()

    def __call__(self, pointcloud):
        if self.distortion_params is not None:
            if random.random() < 0.95:
                for granularity, magnitude in self.distortion_params:
                    pointcloud = self.elastic_distortion(pointcloud, granularity, magnitude)
        return pointcloud


def random_horizontal_flip(coords: torch.Tensor) -> torch.Tensor:
    """dataset/augmentation.py ``RandomHorizontalFlip("z", is_temporal=False)`` on (M, 3) integer voxel coordinates,
    in place: with probability 0.95, for x then y, with probability 0.5 ``c = c.max() - c``.  No host sync."""
    if random.random() < 0.95:
        for axis in (0, 1):
            if random.random() < 0.5:
                c = coords[:, axis]
                coords[:, axis] = c.max() - c
    return coords


def load_gaussian_features(path: str, feature_type: str = "all", device="cuda"):
    """utils/dataset_utils.py ``load_gaussian_ply``: ``(xyz (P,3) fp32, features (P,F) fp32)`` on ``device``, the
    features in PLY property order: ``"all"`` = opacity, f_dc_0..2, f_rest_0..44, scale_0..2, rot_0..3 (56 columns),
    ``"color"`` = f_dc, f_rest (48).  f_rest is channel-major there, unlike ``GaussianModel.get_locs_and_features``,
    so the voxelizer's normal rotation hits columns 3:6 = f_dc_2, f_rest_0, f_rest_1 for ``"all"``, as in the
    reference.  Scenes are SH degree 3, the reference network's 56 / 48 input channels."""
    if feature_type not in ("all", "color"):
        raise ValueError(f"feature_type must be 'all' or 'color', got {feature_type!r}")
    m = load_gaussian_ply(path, GaussianModel(3), device=device)
    P = m._xyz.shape[0]
    dc = m._features_dc.transpose(1, 2).reshape(P, -1)
    rest = m._features_rest.transpose(1, 2).reshape(P, -1)
    parts = [m._opacity, dc, rest, m._scaling, m._rotation] if feature_type == "all" else [dc, rest]
    return m._xyz, torch.cat(parts, dim=1).contiguous()


class FeatureDataset(torch.utils.data.Dataset):
    """dataset/feature_dataset.py ``FeatureDataset`` (same constructor, file discovery and augmentation bounds).
    ``self[i]`` returns ``(locs (M,4) int32 with a leading batch column of ones, features (M,F) fp32, features_gt
    (mask.sum(), C), mask (M,), head_id)``, the tensors on the current CUDA device.  Use with ``num_workers=0``."""

    SCALE_AUGMENTATION_BOUND = (0.9, 1.1)
    ROTATION_AUGMENTATION_BOUND = ((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi))
    TRANSLATION_AUGMENTATION_RATIO_BOUND = ((-0.2, 0.2), (-0.2, 0.2), (0, 0))
    ELASTIC_DISTORT_PARAMS = ((0.2, 0.4), (0.8, 1.6))
    ROTATION_AXIS = "z"

    def __init__(self, gaussians_dir, point_dir, gaussian_iterations=30000, voxel_size=0.02, aug=False,
                 feature_type="all"):
        self.aug = aug
        self.feature_type = feature_type
        self.scenes = sorted(os.listdir(gaussians_dir))
        self.data = []
        for scene in self.scenes:
            for feature in sorted(os.listdir(os.path.join(point_dir, scene))):
                ply_path = os.path.join(gaussians_dir, scene, "point_cloud", f"iteration_{gaussian_iterations}",
                                        "point_cloud.ply")
                self.data.append([ply_path, os.path.join(point_dir, scene, feature), 0])
        self.voxelizer = Voxelizer(voxel_size=voxel_size, clip_bound=None, use_augmentation=aug,
                                   scale_augmentation_bound=self.SCALE_AUGMENTATION_BOUND,
                                   rotation_augmentation_bound=self.ROTATION_AUGMENTATION_BOUND,
                                   translation_augmentation_ratio_bound=self.TRANSLATION_AUGMENTATION_RATIO_BOUND)
        self.elastic = ElasticDistortion(self.ELASTIC_DISTORT_PARAMS)

    def __getitem__(self, index):
        with torch.no_grad():
            ply_path, feature_path, head_id = self.data[index]
            dev = torch.device("cuda", torch.cuda.current_device())
            locs, features = load_gaussian_features(ply_path, self.feature_type, device=dev)
            gt = torch.load(feature_path, map_location="cpu")
            feat, mask_full = gt["feat"].to(dev), gt["mask_full"].to(dev)
            if self.aug:
                locs = self.elastic(locs)
            vox, features, _, _, vox_ind = self.voxelizer.voxelize(locs, features, None, return_ind=True)
            mask, features_gt = distill_targets(vox_ind, mask_full, feat)
            coords = vox.int()
            if self.aug:
                random_horizontal_flip(coords)
            locs = torch.cat([torch.ones((coords.shape[0], 1), dtype=torch.int32, device=dev), coords], dim=1)
        return locs, features, features_gt, mask, head_id

    def __len__(self):
        return len(self.data)


def collate_fn(batch):
    """distill.py:24-30: sample i gets batch index i in column 0 (set in place), then everything is concatenated."""
    locs, features, features_gt, mask, head_id = list(zip(*batch))
    for i in range(len(locs)):
        locs[i][:, 0] *= i
    return torch.cat(locs), torch.cat(features), torch.cat(features_gt), torch.cat(mask), head_id[0]
