"""numpy restatement of the reference's voxelization (dataset/fusion_utils.py: Voxelizer.voxelize without clip_bound,
fnv_hash_vec and sparse_quantize with return_index), written as sgb_voxelize computes it: the transform as
((x T0 + y T1) + z T2) + T3 per axis in fp64 with no fused multiply-add, the floor, the per-axis minimum, FNV-1a 64
over the three uint64 coordinates and a stable unique.  Used by the tests as the checker of the device path."""
from __future__ import annotations

import numpy as np

FNV_OFFSET = np.uint64(14695981039346656037)
FNV_PRIME = np.uint64(1099511628211)


def voxel_floor(xyz: np.ndarray, transform: np.ndarray) -> np.ndarray:
    """(P,3) fp64 floors of xyz under the row-major 3x4 ``transform``."""
    x = np.asarray(xyz).astype(np.float64)
    T = np.asarray(transform, np.float64)[:3, :4]
    # numpy multiplies and adds elementwise with one rounding each: no contraction into an FMA
    return np.floor(((x[:, 0:1] * T[:, 0] + x[:, 1:2] * T[:, 1]) + x[:, 2:3] * T[:, 2]) + T[:, 3])


def fnv_hash(u: np.ndarray) -> np.ndarray:
    """FNV-1a 64 of each row of a (P,3) uint64 array; multiplication wraps modulo 2^64."""
    h = np.full(u.shape[0], FNV_OFFSET, np.uint64)
    with np.errstate(over="ignore"):
        for j in range(u.shape[1]):
            h = (h * FNV_PRIME) ^ u[:, j]
    return h


def voxelize(xyz: np.ndarray, transform: np.ndarray):
    """(first_index (M,) int64, inverse (P,) int64, coords (M,3) int64 origin-aligned, keys (M,) uint64)."""
    v = voxel_floor(xyz, transform)
    if not np.isfinite(v).all():
        raise ValueError("non-finite voxel coordinate")
    u = (v - v.min(0)).astype(np.int64)
    keys = fnv_hash(u.astype(np.uint64))
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    head = np.empty(len(sk), bool)
    head[:1] = True
    head[1:] = sk[1:] != sk[:-1]
    run = np.cumsum(head) - 1
    first = order[head]
    inverse = np.empty(len(keys), np.int64)
    inverse[order] = run
    return first.astype(np.int64), inverse, u[first], sk[head]


def rotate_normals(feats: np.ndarray, rot: np.ndarray) -> np.ndarray:
    """The reference's ``feats[:, 3:6] = feats[:, 3:6] @ M_r[:3, :3].T`` on a copy, in fp64 with the same order
    of operations, rounded back to feats' dtype.  Features of 6 columns or fewer are returned unchanged."""
    out = np.array(feats, copy=True)
    if out.shape[1] > 6:
        n = out[:, 3:6].astype(np.float64)
        R = np.asarray(rot, np.float64)[:3, :3]
        out[:, 3:6] = (n[:, 0:1] * R[:, 0] + n[:, 1:2] * R[:, 1]) + n[:, 2:3] * R[:, 2]
    return out
