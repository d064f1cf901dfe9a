"""Voxelization of Gaussians on the GPU: the reference's ``Voxelizer`` (dataset/fusion_utils.py) with
``sparse_quantize`` computed by ``sgb_voxelize``, bit for bit.

The reference's 3D path (``distill.py``, the ``eval_mink*`` modes of ``eval_segmentation.py``,
``dataset/feature_dataset.py``) copies every scene to the host, voxelizes it with numpy and uploads the result
again.  Here the transform, the hash, the unique and the gathers run on the device; the only host read is the
voxel count M together with the non-finite and overflow status of the call.

Hash collisions between two different voxels merge them, as the reference's FNV-1a ``np.unique`` does: the first
point's coordinates, features and labels stand for both."""
from __future__ import annotations

import collections.abc
import ctypes as C

import numpy as np
import torch
from scipy.linalg import expm

from . import _lib

SGB_E_CUDA, SGB_E_OVERFLOW = -2, -4


def voxel_indices(xyz: torch.Tensor, transform):
    """``sparse_quantize(floor(homo(xyz) @ transform.T), return_index=True)`` of a CUDA (P,3) fp32 or fp64 cloud.

    ``transform``: the first three rows of a 3x4 or 4x4 fp64 matrix.  Returns ``(first_index (M,) int64,
    inverse (P,) int64, coords (M,3) int32)``: np.unique's return_index and return_inverse over the FNV-1a keys, and
    the origin-aligned voxel coordinates of the first points.  Raises ValueError for a non-finite voxel coordinate
    (the reference's result is undefined there) and ``SgbError`` (status -4) when an axis spans 2^31 voxels or
    more.  Enqueued on the current stream; reads M and the status words back once."""
    if not isinstance(xyz, torch.Tensor) or not xyz.is_cuda:
        raise ValueError("xyz must be a CUDA tensor")
    if xyz.dtype not in (torch.float32, torch.float64) or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError(f"xyz must be (P, 3) float32 or float64, got {tuple(xyz.shape)} {xyz.dtype}")
    T = np.ascontiguousarray(np.asarray(transform, np.float64)[:3, :4])
    if T.shape != (3, 4):
        raise ValueError(f"transform must have 3 rows and 4 columns, got {np.asarray(transform).shape}")
    P = xyz.shape[0]
    if not 1 <= P < 2**31:
        raise ValueError(f"need 1 <= P < 2^31 points, got {P}")
    lib = _lib.load()
    dev = xyz.device
    with torch.cuda.device(dev):
        nbytes = lib.sgb_voxelize_workspace_bytes(P)
        if nbytes == 0:
            _lib.check(SGB_E_CUDA, "sgb_voxelize_workspace_bytes")
        x = xyz.contiguous()
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        first = torch.empty(P, dtype=torch.int64, device=dev)
        inverse = torch.empty(P, dtype=torch.int64, device=dev)
        coords = torch.empty((P, 3), dtype=torch.int32, device=dev)
        counts = torch.empty(3, dtype=torch.int64, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        name = "sgb_voxelize_f64" if x.dtype == torch.float64 else "sgb_voxelize"
        _lib.check(getattr(lib, name)(P, x.data_ptr(), (C.c_double * 12)(*T.ravel()), ws.data_ptr(), first.data_ptr(),
                                      inverse.data_ptr(), coords.data_ptr(), counts.data_ptr(), stream), name)
        M, nonfinite, status = counts.tolist()
    if nonfinite:
        raise ValueError(f"{nonfinite} of {P} points have a non-finite voxel coordinate")
    if status != 0:
        raise _lib.SgbError(f"sgb_voxelize: the cloud spans 2^31 voxels or more on an axis; the int32 voxel "
                            f"coordinates cannot hold it (status {status})")
    return first[:M], inverse, coords[:M]


def _rotate_normals(feats, rot):
    """``feats[:, 3:6] @ rot[:3, :3].T`` in fp64, rounded to feats' dtype (fusion_utils.py:203-204), on a copy for
    numpy and in place for a tensor the caller owns.  The products and sums are rounded one at a time, in the
    order numpy's 3x3 product takes them, so the result is bitwise the reference's."""
    if feats.shape[1] <= 6:
        return feats
    R = np.asarray(rot, np.float64)[:3, :3]
    if isinstance(feats, torch.Tensor):
        R = torch.as_tensor(R, device=feats.device)
        n = feats[:, 3:6].double()
        feats[:, 3:6] = ((n[:, 0:1] * R[:, 0] + n[:, 1:2] * R[:, 1]) + n[:, 2:3] * R[:, 2]).to(feats.dtype)
    else:
        n = feats[:, 3:6].astype(np.float64)
        feats[:, 3:6] = (n[:, 0:1] * R[:, 0] + n[:, 1:2] * R[:, 1]) + n[:, 2:3] * R[:, 2]
    return feats


class Voxelizer:
    """The reference's ``Voxelizer`` (same constructor and results) with the quantization on the GPU.

    numpy inputs give numpy outputs (coords as float64, as the reference returns them); CUDA tensors give CUDA
    tensors and are never copied to the host.  Coordinates are float32 (the Gaussians' xyz) or float64 (the cloud
    after ``feature_dataset.ElasticDistortion``).  ``clip_bound`` is not supported: no reference caller sets it."""

    def __init__(self, voxel_size=1, clip_bound=None, use_augmentation=False, scale_augmentation_bound=None,
                 rotation_augmentation_bound=None, translation_augmentation_ratio_bound=None, ignore_label=255):
        if clip_bound is not None:
            raise NotImplementedError("Voxelizer: clip_bound is not supported")
        self.voxel_size = voxel_size
        self.clip_bound = clip_bound
        self.ignore_label = ignore_label
        self.use_augmentation = use_augmentation
        self.scale_augmentation_bound = scale_augmentation_bound
        self.rotation_augmentation_bound = rotation_augmentation_bound
        self.translation_augmentation_ratio_bound = translation_augmentation_ratio_bound

    def get_transformation_matrix(self):
        """``(voxelization_matrix, rotation_matrix)``, 4x4 fp64 each, drawn from ``np.random`` in the reference's
        order: one angle per bounded axis (x, y, z), a shuffle of the three axis rotations, then the scale."""
        voxelization, rotation = np.eye(4), np.eye(4)
        rot = np.eye(3)
        if self.use_augmentation and self.rotation_augmentation_bound is not None:
            if not isinstance(self.rotation_augmentation_bound, collections.abc.Iterable):
                raise ValueError("rotation_augmentation_bound must be a sequence of per-axis bounds")
            mats = []
            for axis_index, bound in enumerate(self.rotation_augmentation_bound):
                axis = np.zeros(3)
                axis[axis_index] = 1
                theta = np.random.uniform(*bound) if bound is not None else 0
                # rotation by theta about the unit axis: exp of its cross-product matrix
                mats.append(expm(np.cross(np.eye(3), axis / np.linalg.norm(axis) * theta)))
            np.random.shuffle(mats)
            rot = mats[0] @ mats[1] @ mats[2]
        rotation[:3, :3] = rot
        scale = 1 / self.voxel_size
        if self.use_augmentation and self.scale_augmentation_bound is not None:
            scale *= np.random.uniform(*self.scale_augmentation_bound)
        np.fill_diagonal(voxelization[:3, :3], scale)
        return voxelization, rotation

    def voxelize(self, coords, feats, labels, center=None, link=None, return_ind=False):
        """``(coords, feats, labels, inverse)``, then ``first_index`` with ``return_ind`` or ``link[first_index]``
        with a ``link``, as the reference returns them.  ``center`` only matters with a clip bound."""
        if coords.ndim != 2 or coords.shape[1] != 3 or coords.shape[0] == 0 or feats.shape[0] != coords.shape[0]:
            raise ValueError(f"need coords (P, 3) with P > 0 and feats with P rows, got {tuple(coords.shape)} and "
                             f"{tuple(feats.shape)}")
        if coords.dtype not in (np.float32, np.float64, torch.float32, torch.float64):
            raise ValueError(f"coords must be float32 or float64, got {coords.dtype}")
        M_v, M_r = self.get_transformation_matrix()
        transform = M_r @ M_v if self.use_augmentation else M_v
        if isinstance(coords, torch.Tensor):
            first, inverse, vox = voxel_indices(coords, transform)
            out_feats = _rotate_normals(feats.index_select(0, first), M_r)
            out = [vox.double(), out_feats, None if labels is None else labels[first], inverse]
        else:
            xyz = torch.from_numpy(np.ascontiguousarray(coords)).cuda()
            first_t, inverse_t, vox_t = voxel_indices(xyz, transform)
            first = first_t.cpu().numpy()
            out = [vox_t.cpu().numpy().astype(np.float64), _rotate_normals(feats[first], M_r),
                   None if labels is None else labels[first], inverse_t.cpu().numpy()]
        if return_ind:
            return (*out, first)
        if link is not None:
            return (*out, link[first])
        return tuple(out)


def voxelize_gaussians(gaussians, voxel_size, feature_type="all"):
    """What ``eval_mink`` / ``distill.py`` hand to ``ME.SparseTensor``, computed on the device:
    ``(locs (M,4) int32 with a leading batch column of ones, features (M,F) fp32, vox_ind (M,) int64)``.
    ``vox_ind`` are the Gaussians that stand for the voxels (``_features_semantic[vox_ind] = output``).  Equal to
    ``Voxelizer(voxel_size).voxelize(*gaussians.get_locs_and_features(feature_type), None, return_ind=True)``."""
    xyz, feats = gaussians.get_locs_and_features(feature_type, device=True)
    M_v, M_r = Voxelizer(voxel_size).get_transformation_matrix()
    first, _, vox = voxel_indices(xyz, M_v)
    features = _rotate_normals(feats.index_select(0, first).float(), M_r)
    locs = torch.cat([torch.ones((vox.shape[0], 1), dtype=torch.int32, device=vox.device), vox], dim=1)
    return locs, features, first


def distill_targets(vox_ind: torch.Tensor, mask_full: torch.Tensor, feat: torch.Tensor):
    """``(mask, features_gt)`` of dataset/feature_dataset.py:74-88 on the device: ``mask = mask_full[vox_ind]``
    and, for the voxels whose Gaussian is masked, the rows of ``feat`` (one row per masked Gaussian, in Gaussian
    order) that belong to them."""
    if not (vox_ind.device == mask_full.device == feat.device):
        raise ValueError("vox_ind, mask_full and feat must be on one device")
    mask = mask_full[vox_ind]
    valid = mask_full != 0
    rank = torch.cumsum(valid, dim=0) - 1            # row of each masked Gaussian in feat
    features_gt = feat[rank[vox_ind[valid[vox_ind]]]]
    return mask, features_gt
