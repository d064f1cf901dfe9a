"""CPU: the numpy voxelization oracle against fixtures of the reference's own Voxelizer
(tests/golden/make_voxel_golden.py), the random draws of Voxelizer.get_transformation_matrix, the FNV-1a loop, and
argument validation of sgb_voxelize, which runs before any CUDA call."""
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
from semantic_gaussians_b200.voxelize import Voxelizer  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "voxel_golden.npz"))


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_reference_voxelizer(case):
    xyz, feats = voxel_inputs(case)
    M_v, M_r = GOLDEN[f"{case}_M_v"], GOLDEN[f"{case}_M_r"]
    transform = M_r @ M_v if CASES[case][4] else M_v
    first, inverse, coords, _ = vo.voxelize(xyz, transform)
    assert np.array_equal(first, GOLDEN[f"{case}_inds"])
    assert np.array_equal(inverse, GOLDEN[f"{case}_inds_reconstruct"])
    assert np.array_equal(digest(coords.astype(np.float64)), GOLDEN[f"{case}_coords.sha256"])
    assert np.array_equal(digest(vo.rotate_normals(feats[first], M_r)), GOLDEN[f"{case}_feats.sha256"])


@pytest.mark.parametrize("case", sorted(CASES))
def test_transformation_matrix_draws_like_the_reference(case):
    np.random.seed(CASES[case][0])
    M_v, M_r = Voxelizer(**voxelizer_kwargs(case)).get_transformation_matrix()
    assert M_v.dtype == M_r.dtype == np.float64
    assert np.array_equal(M_v, GOLDEN[f"{case}_M_v"]) and np.array_equal(M_r, GOLDEN[f"{case}_M_r"])


def test_clip_bound_is_not_supported():
    with pytest.raises(NotImplementedError):
        Voxelizer(0.02, clip_bound=((-1, 1), (-1, 1), (-1, 1)))


def _fnv_int(row):
    h = 14695981039346656037
    for u in row:
        h = ((h * 1099511628211) % 2**64) ^ u
    return h


def test_fnv_hash_on_hand_picked_coordinates():
    rows = [(0, 0, 0), (1, 0, 0), (0, 0, 1), (0, 1, 0), (2**31 - 1, 2**31 - 1, 2**31 - 1), (7, 2**40, 3),
            (2**64 - 1, 0, 2**63), (123456789, 987654321, 5)]
    got = vo.fnv_hash(np.array(rows, dtype=np.uint64))
    assert [int(h) for h in got] == [_fnv_int(r) for r in rows]
    # the offset basis times the prime wraps: the key of the origin is not the product over the integers
    assert _fnv_int((0, 0, 0)) == (14695981039346656037 * 1099511628211 ** 3) % 2**64
    assert int(got[0]) == 0xD94D12186C0F2FB7


FMA_X, FMA_T0, FMA_T3 = 0.9491629600524902, 26.338996623527596, -25.0


def test_oracle_floor_is_unfused_fp64():
    """((x T0 + y T1) + z T2) + T3 rounded step by step: x T0 lies just below 25 and rounds to 25.0, so the
    unfused sum is 0 while an FMA would keep the deficit and floor to -1."""
    from fractions import Fraction
    assert float(np.float32(FMA_X)) == FMA_X and FMA_X * FMA_T0 == 25.0
    assert Fraction(FMA_X) * Fraction(FMA_T0) < 25
    T = np.zeros((3, 4))
    T[:, 0], T[:, 3] = FMA_T0, FMA_T3
    v = vo.voxel_floor(np.array([[FMA_X, 0, 0]], np.float32), T)
    assert (v == 0.0).all()


def test_workspace_bytes_refuses_point_counts_out_of_range():
    lib = _lib.load()
    for P in (0, -1, 2**31, 2**40):
        assert lib.sgb_voxelize_workspace_bytes(P) == 0


def _args():
    xyz = (C.c_float * 6)()
    buf = (C.c_int64 * 64)()
    base = C.addressof(buf)
    base += (-base) % 16
    return dict(P=2, xyz=C.addressof(xyz), transform=(C.c_double * 12)(), workspace=base, first_index=base,
                inverse=base, coords=base, counts=base)


@pytest.mark.parametrize("kw,msg", [
    (dict(P=0), b"P = 0"),
    (dict(P=-3), b"P = -3"),
    (dict(P=2**31), b"exceeds"),
    (dict(xyz=None), b"null xyz"),
    (dict(transform=None), b"null transform"),
    (dict(workspace=None), b"null workspace"),
    (dict(workspace="misaligned"), b"not 16-byte aligned"),
    (dict(first_index=None), b"null first_index"),
    (dict(inverse=None), b"null first_index / inverse / coords"),
    (dict(coords=None), b"null first_index / inverse / coords"),
    (dict(counts=None), b"null counts"),
])
def test_voxelize_argument_validation_happens_before_cuda(kw, msg):
    lib = _lib.load()
    a = _args()
    if kw.get("workspace") == "misaligned":
        kw = dict(workspace=a["workspace"] + 8)
    a.update(kw)
    rc = lib.sgb_voxelize(a["P"], a["xyz"], a["transform"], a["workspace"], a["first_index"], a["inverse"],
                          a["coords"], a["counts"], None)
    assert rc == -1
    assert msg in lib.sgb_last_error()


def _cpu_model(P=50, seed=0):
    g = torch.Generator().manual_seed(seed)
    m = GaussianModel(3)
    m._xyz = torch.randn(P, 3, generator=g)
    m._opacity = torch.randn(P, 1, generator=g)
    m._features_dc = torch.randn(P, 1, 3, generator=g)
    m._features_rest = torch.randn(P, 15, 3, generator=g)
    m._scaling = torch.randn(P, 3, generator=g)
    m._rotation = torch.randn(P, 4, generator=g)
    return m


@pytest.mark.parametrize("feature_type,parts,F", [
    ("all", ("_opacity", "_features_dc", "_features_rest", "_scaling", "_rotation"), 56),
    ("color", ("_features_dc", "_features_rest"), 48),
])
def test_get_locs_and_features_is_the_reference_concatenation(feature_type, parts, F):
    m = _cpu_model()
    locs, feats = m.get_locs_and_features(feature_type)
    assert isinstance(locs, np.ndarray) and locs.dtype == np.float32 and np.array_equal(locs, m._xyz.numpy())
    want = np.concatenate([getattr(m, p).numpy().reshape(50, -1) for p in parts], axis=-1)
    assert feats.shape == (50, F) and feats.dtype == np.float32 and np.array_equal(feats, want)
    locs[0, 0] = 1e9                                        # a copy, as the reference's .clone().cpu().numpy()
    assert m._xyz[0, 0] != 1e9
    with pytest.raises(ValueError):
        m.get_locs_and_features("semantic")
