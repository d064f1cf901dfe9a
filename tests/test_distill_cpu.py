"""CPU: the 3D distillation sample and loss that need no device.  The numpy restatement of the elastic-distortion
lookup (oracle/augment_oracle.py) is bitwise the reference's ElasticDistortion (tests/golden/distill_golden.npz),
the PLY loader's column order is the reference's, and every new entry point rejects bad arguments before any CUDA
call."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_distill_golden import ELASTIC_CASES, ELASTIC_PARAMS, elastic_input, seed_all  # noqa: E402
from make_raster_golden import digest  # noqa: E402

from oracle import augment_oracle as ao  # noqa: E402
from semantic_gaussians_b200 import _lib, semantic  # noqa: E402
from semantic_gaussians_b200.feature_dataset import ElasticDistortion, load_gaussian_features  # noqa: E402
from semantic_gaussians_b200.io_formats import gaussian_attribute_names, write_vertex_ply  # noqa: E402
from semantic_gaussians_b200.voxelize import Voxelizer  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "distill_golden.npz"))


@pytest.mark.parametrize("case", sorted(ELASTIC_CASES))
def test_oracle_elastic_distortion_is_reference_golden(case):
    xyz = elastic_input(case)
    seed_all(ELASTIC_CASES[case][0])
    got, dims = ao.elastic_distortion_all(xyz, ELASTIC_PARAMS)
    assert np.array_equal(np.asarray(dims, np.int64).reshape(-1, 3), GOLDEN[f"{case}_noise_dims"])
    if not dims:                       # the gate skipped: the input comes back as it is
        got = xyz
    assert np.array_equal(digest(got), GOLDEN[f"{case}_xyz.sha256"])


def test_oracle_lookup_outside_and_nan():
    noise = np.arange(3 * 3 * 3 * 3, dtype=np.float32).reshape(3, 3, 3, 3)
    ax = [np.array([0.0, 1.0, 2.0])] * 3
    xyz = np.array([[0.5, 0.5, 0.5], [-0.1, 1, 1], [1, 1, 2.5], [np.nan, 1, 1], [2.0, 2.0, 2.0], [-0.0, 0, 0]])
    out = ao.lookup(xyz, noise, ax, 2.0)
    # the trilinear value at the centre of the first cell is the mean of its 8 corners
    corners = noise[:2, :2, :2].reshape(-1, 3).astype(np.float64)
    assert np.allclose(out[0], 0.5 + corners.mean(0) * 2.0)
    assert np.array_equal(out[1], xyz[1]) and np.array_equal(out[2], xyz[2])
    assert np.isnan(out[3]).all()
    assert np.array_equal(out[4], 2.0 + noise[2, 2, 2].astype(np.float64) * 2.0)   # the closed upper end
    assert np.array_equal(out[5], noise[0, 0, 0].astype(np.float64) * 2.0)


@pytest.mark.parametrize("feature_type", ["all", "color"])
def test_ply_columns_are_reference_property_order(tmp_path, feature_type):
    names = gaussian_attribute_names(3, 45)
    P = 4
    table = (np.arange(len(names), dtype=np.float32)[None, :] + 1000 * np.arange(P, dtype=np.float32)[:, None])
    path = str(tmp_path / "point_cloud.ply")
    write_vertex_ply(path, names, table)
    xyz, feats = load_gaussian_features(path, feature_type, device="cpu")
    col = {n: table[:, i] for i, n in enumerate(names)}
    # utils/dataset_utils.py load_gaussian_ply: opacity, f_dc_0..2, f_rest_0..44 by index, scale_*, rot_*
    order = ([f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(45)])
    if feature_type == "all":
        order = ["opacity"] + order + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)]
    assert feats.dtype == torch.float32 and feats.shape == (P, len(order))
    assert np.array_equal(feats.numpy(), np.stack([col[n] for n in order], axis=1))
    assert np.array_equal(xyz.numpy(), table[:, :3])
    # the voxelizer's normal rotation takes columns 3:6
    want = ["f_dc_2", "f_rest_0", "f_rest_1"] if feature_type == "all" else ["f_rest_0", "f_rest_1", "f_rest_2"]
    assert [order[i] for i in range(3, 6)] == want


def test_elastic_displace_rejects_bad_arguments():
    lib = _lib.load()
    ok = dict(P=10, xyz=8, f64=0, grid=8, nx=3, ny=3, nz=3, axes=8, mag=0.4, out=16)

    def call(**kw):
        a = {**ok, **kw}
        return lib.sgb_elastic_displace(a["P"], a["xyz"], a["f64"], a["grid"], a["nx"], a["ny"], a["nz"], a["axes"],
                                        C.c_double(a["mag"]), a["out"], None)
    for kw, msg in ((dict(P=0), b"P = 0"), (dict(P=2**31), b"P = 2147483648"), (dict(f64=2), b"xyz_is_f64"),
                    (dict(ny=1), b"at least 2 nodes"), (dict(nx=2000, ny=2000, nz=2000), b"exceeds"),
                    (dict(xyz=None), b"null"), (dict(grid=None), b"null"), (dict(axes=None), b"null"),
                    (dict(out=None), b"null"), (dict(out=8), b"alias")):
        assert call(**kw) == -1, kw
        assert msg in lib.sgb_last_error(), (kw, lib.sgb_last_error())


def test_voxel_feature_loss_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.sgb_voxel_feature_loss_workspace_bytes(-1) == 0
    assert lib.sgb_voxel_feature_loss_workspace_bytes(2**31) == 0
    ok = dict(M=100, F=1536, out=256, mask=256, K=10, C=768, head=1, y=256, dt=0, lt=0, grad=256, ws=256, loss=256)

    def call(**kw):
        a = {**ok, **kw}
        return lib.sgb_voxel_feature_loss(a["M"], a["F"], a["out"], a["mask"], a["K"], a["C"], a["head"], a["y"],
                                          a["dt"], a["lt"], a["grad"], a["ws"], a["loss"], None)
    for kw, msg in ((dict(M=-1), b"M = -1"), (dict(M=2**31), b"M = 2147483648"), (dict(C=0), b"C = 0"),
                    (dict(C=1025, F=4096, head=0), b"C = 1025"), (dict(head=2), b"does not fit"),
                    (dict(head=-1), b"does not fit"), (dict(K=101), b"K = 101"), (dict(K=-1), b"K = -1"),
                    (dict(dt=2), b"target_dtype"), (dict(lt=3), b"loss_type"), (dict(loss=None), b"null loss"),
                    (dict(out=None), b"null output"), (dict(mask=None), b"null output"),
                    (dict(grad=None), b"null output"), (dict(y=None), b"null target"),
                    (dict(ws=None), b"null workspace"), (dict(ws=258), b"16-byte")):
        assert call(**kw) == -1, kw
        assert msg in lib.sgb_last_error(), (kw, lib.sgb_last_error())


def test_voxelize_f64_rejects_bad_arguments():
    lib = _lib.load()
    T = (C.c_double * 12)()
    assert lib.sgb_voxelize_f64(0, 8, T, 256, 8, 8, 8, 8, None) == -1
    assert b"sgb_voxelize_f64: P = 0" in lib.sgb_last_error()
    assert lib.sgb_voxelize_f64(5, None, T, 256, 8, 8, 8, 8, None) == -1
    assert b"null xyz" in lib.sgb_last_error()


def test_python_entry_points_reject_cpu_and_bad_inputs():
    with pytest.raises(ValueError, match="CUDA"):
        semantic.voxel_feature_loss_and_grad(torch.zeros(4, 768), torch.ones(4, dtype=torch.bool),
                                             torch.zeros(4, 768))
    with pytest.raises(ValueError, match="numpy array or a CUDA tensor"):
        ElasticDistortion(ELASTIC_PARAMS).elastic_distortion(torch.zeros(4, 3), 0.2, 0.4)
    with pytest.raises(ValueError, match="float32 or float64"):
        Voxelizer(0.02).voxelize(np.zeros((4, 3), np.float16), np.zeros((4, 8), np.float32), None)
