"""GPU: sgb_voxelize and the Voxelizer built on it, bit for bit against the reference's own Voxelizer
(tests/golden/voxel_golden.npz) and the numpy oracle (oracle/voxel_oracle.py), plus the status words, determinism,
voxelize_gaussians and distill_targets."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_raster_golden import digest  # noqa: E402
from make_voxel_golden import CASES, voxel_inputs, voxelizer_kwargs  # noqa: E402

from oracle import voxel_oracle as vo  # noqa: E402
from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.voxelize import Voxelizer, distill_targets, voxel_indices, voxelize_gaussians  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "voxel_golden.npz"))
DEV = "cuda"


def _abi(xyz_np, transform):
    """sgb_voxelize called directly: (first_index, inverse, coords, counts) of the full P-sized buffers."""
    lib = _lib.load()
    P = len(xyz_np)
    xyz = torch.from_numpy(np.ascontiguousarray(xyz_np, np.float32)).to(DEV)
    ws = torch.empty(lib.sgb_voxelize_workspace_bytes(P), dtype=torch.uint8, device=DEV)
    first = torch.full((P,), -7, dtype=torch.int64, device=DEV)
    inverse = torch.empty(P, dtype=torch.int64, device=DEV)
    coords = torch.empty((P, 3), dtype=torch.int32, device=DEV)
    counts = torch.full((3,), -7, dtype=torch.int64, device=DEV)
    T = (C.c_double * 12)(*np.asarray(transform, np.float64)[:3, :4].ravel())
    rc = lib.sgb_voxelize(P, xyz.data_ptr(), T, ws.data_ptr(), first.data_ptr(), inverse.data_ptr(),
                          coords.data_ptr(), counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.sgb_last_error()
    return first.cpu().numpy(), inverse.cpu().numpy(), coords.cpu().numpy(), counts.cpu().numpy()


def _check_against_oracle(xyz, transform):
    first, inverse, coords, counts = _abi(xyz, transform)
    M = counts[0]
    want_first, want_inverse, want_coords, _ = vo.voxelize(xyz, transform)
    assert list(counts) == [len(want_first), 0, 0]
    assert np.array_equal(first[:M], want_first)
    assert np.array_equal(inverse, want_inverse)
    assert np.array_equal(coords[:M], want_coords)


def _golden_transform(case):
    M_v, M_r = GOLDEN[f"{case}_M_v"], GOLDEN[f"{case}_M_r"]
    return M_v, M_r, (M_r @ M_v if CASES[case][4] else M_v)


@pytest.mark.parametrize("case", sorted(CASES))
def test_abi_matches_reference_golden(case):
    xyz, _ = voxel_inputs(case)
    _, _, transform = _golden_transform(case)
    first, inverse, coords, counts = _abi(xyz, transform)
    M = counts[0]
    assert counts[1] == 0 and counts[2] == 0
    assert np.array_equal(first[:M], GOLDEN[f"{case}_inds"])
    assert np.array_equal(inverse, GOLDEN[f"{case}_inds_reconstruct"])
    assert np.array_equal(digest(coords[:M].astype(np.float64)), GOLDEN[f"{case}_coords.sha256"])


@pytest.mark.parametrize("on_device", [False, True], ids=["numpy", "cuda"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_voxelizer_matches_reference_golden(case, on_device):
    xyz, feats = voxel_inputs(case)
    labels = np.arange(len(xyz)) * 3
    if on_device:
        xyz, feats, labels = (torch.from_numpy(a).to(DEV) for a in (xyz, feats, labels))
    np.random.seed(CASES[case][0])
    coords, f, lab, inverse, inds = Voxelizer(**voxelizer_kwargs(case)).voxelize(xyz, feats, labels,
                                                                                return_ind=True)
    if on_device:
        assert all(t.is_cuda for t in (coords, f, lab, inverse, inds))
        coords, f, lab, inverse, inds = (t.cpu().numpy() for t in (coords, f, lab, inverse, inds))
    assert coords.dtype == np.float64 and f.dtype == np.float32 and inds.dtype == inverse.dtype == np.int64
    assert np.array_equal(inds, GOLDEN[f"{case}_inds"])
    assert np.array_equal(inverse, GOLDEN[f"{case}_inds_reconstruct"])
    assert np.array_equal(digest(coords), GOLDEN[f"{case}_coords.sha256"])
    assert np.array_equal(digest(f), GOLDEN[f"{case}_feats.sha256"])
    assert np.array_equal(lab, inds * 3)


def test_voxelizer_return_forms():
    xyz, feats = voxel_inputs("plain_002")
    before = feats.copy()
    vox = Voxelizer(0.02)
    c, f, lab, inv = vox.voxelize(xyz, feats, None)
    c2, f2, lab2, inv2, link = vox.voxelize(xyz, feats, None, link=np.arange(len(xyz)) + 5)
    assert lab is None and lab2 is None
    assert np.array_equal(c, c2) and np.array_equal(f, f2) and np.array_equal(inv, inv2)
    assert np.array_equal(link - 5, GOLDEN["plain_002_inds"])
    assert np.array_equal(feats, before)                     # the input features are not rotated in place


def _cloud(kind, P, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "one_voxel":
        return rng.uniform(0.205, 0.215, (P, 3)).astype(np.float32), np.diag([50.0, 50.0, 50.0, 1.0])
    if kind == "distinct":              # voxel centres of a 128 x 128 x 64 grid, shuffled
        i = rng.permutation(P)
        xyz = np.stack([i % 128, (i // 128) % 128, i // 16384], 1) + 0.5
        return xyz.astype(np.float32), np.eye(4)
    if kind == "duplicates":            # a handful of points repeated exactly
        base = rng.uniform(-1, 1, (max(P // 50, 1), 3)).astype(np.float32)
        return base[rng.integers(0, len(base), P)], np.diag([50.0, 50.0, 50.0, 1.0])
    # a wide cloud under a rotation: about 2e9 voxels along x, close to the int32 limit
    xyz = rng.uniform(-1e6, 1e6, (P, 3)).astype(np.float32)
    np.random.seed(seed)
    M_v, M_r = Voxelizer(1.1e-3, use_augmentation=True, rotation_augmentation_bound=((0, 0), (0, 0), (-0.01, 0.01)),
                         scale_augmentation_bound=(0.9, 1.1)).get_transformation_matrix()
    return xyz, M_r @ M_v


@pytest.mark.parametrize("P", [1, 2, 1000, 2**16 + 3, 1 << 20])
@pytest.mark.parametrize("kind", ["one_voxel", "distinct", "duplicates", "large_extent"])
def test_abi_matches_oracle(kind, P):
    xyz, transform = _cloud(kind, P)
    _check_against_oracle(xyz, transform)


def test_floor_is_not_contracted_into_an_fma():
    """x T0 lies just below 25 and rounds to 25.0: unfused, the point is 25 voxels from the origin point; an FMA
    would put it at 24."""
    T = np.zeros((3, 4))
    T[:, 0], T[:, 3] = 26.338996623527596, -25.0
    xyz = np.array([[0.9491629600524902, 0, 0], [0, 0, 0]], np.float32)
    first, inverse, coords, counts = _abi(xyz, T)
    assert counts[0] == 2 and sorted(coords[:2].tolist()) == [[0, 0, 0], [25, 25, 25]]
    _check_against_oracle(xyz, T)


@pytest.mark.parametrize("span,overflow", [(2**31 - 128, False), (2**31, True), (3.0e38, True)])
def test_extent_of_2_31_voxels_overflows(span, overflow):
    xyz = np.array([[0, 0, 0], [span, 1, 2], [5, 5, 5]], np.float32)
    _, _, coords, counts = _abi(xyz, np.eye(4))
    assert counts[1] == 0 and counts[2] == (-4 if overflow else 0)
    if overflow:
        with pytest.raises(_lib.SgbError, match=r"status -4"):
            voxel_indices(torch.from_numpy(xyz).to(DEV), np.eye(4))
    else:
        assert coords[:counts[0]].max() == 2**31 - 128


def test_non_finite_points_are_counted_and_raise():
    xyz = np.array([[0, 0, 0], [np.nan, 1, 2], [1, np.inf, 0], [2, 2, 2]], np.float32)
    _, _, _, counts = _abi(xyz, np.eye(4))
    assert counts[1] == 2
    with pytest.raises(ValueError, match="non-finite"):
        Voxelizer(0.02).voxelize(torch.from_numpy(xyz).to(DEV), torch.zeros(4, 8, device=DEV), None)
    # finite input, non-finite product
    _, _, _, counts = _abi(np.array([[3e38, 0, 0], [0, 0, 0]], np.float32), np.diag([1e300, 1, 1, 1]))
    assert counts[1] == 1


def test_two_calls_give_identical_output():
    xyz, transform = _cloud("large_extent", 300_000, seed=3)
    a, b = _abi(xyz, transform), _abi(xyz, transform)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def _model(P, seed=0):
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((P, 4))
    m = GaussianModel.from_activated(
        xyz=rng.uniform(-2, 2, (P, 3)), scales=np.exp(rng.standard_normal((P, 3)) - 4),
        rotations=q / np.linalg.norm(q, axis=1, keepdims=True), opacity=rng.uniform(0.05, 0.95, P),
        shs=rng.standard_normal((P, 16, 3)), device=DEV)
    return m


@pytest.mark.parametrize("feature_type,F", [("all", 56), ("color", 48)])
def test_voxelize_gaussians_equals_voxelizer_on_locs_and_features(feature_type, F):
    m = _model(200_000)
    locs, features, vox_ind = voxelize_gaussians(m, 0.02, feature_type)
    assert locs.dtype == torch.int32 and features.dtype == torch.float32 and vox_ind.dtype == torch.int64
    assert locs.shape[1] == 4 and features.shape[1] == F and (locs[:, 0] == 1).all()
    np_locs, np_feats = m.get_locs_and_features(feature_type)
    dev_locs, dev_feats = m.get_locs_and_features(feature_type, device=True)
    assert dev_locs.is_cuda and torch.equal(dev_feats.cpu(), torch.from_numpy(np_feats))
    c, f, _, _, ind = Voxelizer(0.02).voxelize(np_locs, np_feats, None, return_ind=True)
    assert np.array_equal(locs[:, 1:].cpu().numpy(), c.astype(np.int32))
    assert np.array_equal(features.cpu().numpy(), f) and np.array_equal(vox_ind.cpu().numpy(), ind)
    first, _, coords, _ = vo.voxelize(np_locs, np.diag([50.0, 50.0, 50.0, 1.0]))
    assert np.array_equal(ind, first) and np.array_equal(c, coords)


def _reference_distill_targets(vox_ind, mask_chunk, features_gt):
    """dataset/feature_dataset.py:74-88 as written there, on CPU tensors."""
    mask = mask_chunk[vox_ind]
    mask_ind = mask_chunk.nonzero(as_tuple=False)[:, 0]
    index1 = -torch.ones(mask_chunk.shape[0], dtype=int)
    index1[mask_ind] = mask_ind
    index1 = index1[vox_ind]
    chunk_ind = index1[index1 != -1]
    index2 = torch.zeros(mask_chunk.shape[0])
    index2[mask_ind] = 1
    index3 = torch.cumsum(index2, dim=0, dtype=int)
    indices = index3[chunk_ind] - 1
    return mask, features_gt[indices]


@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.uint8])
def test_distill_targets_equals_feature_dataset(mask_dtype):
    m = _model(100_000, seed=1)
    _, _, vox_ind = voxelize_gaussians(m, 0.05)
    g = torch.Generator().manual_seed(0)
    mask_full = (torch.rand(100_000, generator=g) < 0.6).to(mask_dtype)
    feat = torch.randn(int(mask_full.sum()), 16, generator=g).half()
    want_mask, want_feat = _reference_distill_targets(vox_ind.cpu(), mask_full, feat)
    mask, got = distill_targets(vox_ind, mask_full.to(DEV), feat.to(DEV))
    assert mask.dtype == mask_dtype and torch.equal(mask.cpu(), want_mask)
    assert got.dtype == feat.dtype and torch.equal(got.cpu(), want_feat)
