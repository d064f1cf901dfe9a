"""CPU: on-disk formats — Gaussian PLY in the reference's vertex layout, fused-feature .pt."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from semantic_gaussians_b200 import io_formats as io
from semantic_gaussians_b200.gaussian_model import GaussianModel


def _model(n=37, deg=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    m = GaussianModel(deg)
    m._xyz = torch.randn(n, 3, generator=g)
    m._features_dc = torch.randn(n, 1, 3, generator=g)
    m._features_rest = torch.randn(n, (deg + 1) ** 2 - 1, 3, generator=g)
    m._opacity = torch.randn(n, 1, generator=g)
    m._scaling = torch.randn(n, 3, generator=g)
    m._rotation = torch.randn(n, 4, generator=g)
    return m


def test_ply_header_and_layout_match_the_reference_writer(tmp_path):
    m = _model()
    p = str(tmp_path / "point_cloud" / "iteration_1" / "point_cloud.ply")
    m.save_ply(p)
    raw = open(p, "rb").read()
    names = io.gaussian_attribute_names(3, 45)
    assert names[:9] == ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"]
    assert names[9] == "f_rest_0" and names[54:] == ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 37\n" +
              "".join(f"property float {n}\n" for n in names) + "end_header\n").encode()
    assert raw.startswith(header) and len(raw) == len(header) + 37 * 62 * 4       # plyfile's byte layout
    row0 = np.frombuffer(raw[len(header):len(header) + 62 * 4], dtype="<f4")
    assert np.array_equal(row0[:3], m._xyz[0].numpy()) and np.all(row0[3:6] == 0)
    assert np.array_equal(row0[6:9], m._features_dc[0, 0].numpy())
    # f_rest is channel-major: f_rest_k = rest[:, k % 15, k // 15]  (transpose(1,2).flatten, gaussian_model.py:271)
    assert np.array_equal(row0[9:24], m._features_rest[0, :, 0].numpy())
    assert row0[54] == m._opacity[0, 0] and np.array_equal(row0[58:62], m._rotation[0].numpy())


def test_ply_round_trip_and_reader_variants(tmp_path):
    m = _model(50, 3, 1)
    p = str(tmp_path / "a.ply")
    m.save_ply(p)
    r = GaussianModel(3)
    r.load_ply(p, device="cpu")
    for k in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"):
        assert torch.equal(getattr(r, k), getattr(m, k)), k
    assert r.active_sh_degree == 3 and r._features_rest.shape == (50, 15, 3)
    # big-endian and ascii bodies, shuffled property order, comments
    el = io.read_vertex_ply(p)
    names = list(el)[::-1]
    tab = np.stack([el[n] for n in names], axis=1)
    hdr = "ply\nformat binary_big_endian 1.0\ncomment x\nelement vertex 50\n" + "".join(f"property float32 {n}\n" for n in names) + "end_header\n"
    open(tmp_path / "be.ply", "wb").write(hdr.encode() + tab.astype(">f4").tobytes())
    hdr = "ply\nformat ascii 1.0\nelement vertex 50\n" + "".join(f"property double {n}\n" for n in names) + "end_header\n"
    open(tmp_path / "as.ply", "w").write(hdr + "\n".join(" ".join(repr(float(v)) for v in row) for row in tab) + "\n")
    for q in ("be.ply", "as.ply"):
        r2 = GaussianModel(3)
        r2.load_ply(str(tmp_path / q), device="cpu")
        assert torch.equal(r2._xyz, m._xyz) and torch.equal(r2._features_rest, m._features_rest)
    with pytest.raises(ValueError):
        GaussianModel(2).load_ply(p, device="cpu")                     # SH degree mismatch (:307 assert)
    open(tmp_path / "bad.ply", "wb").write(b"plx\n")
    with pytest.raises(ValueError):
        io.read_vertex_ply(str(tmp_path / "bad.ply"))


def test_fused_feature_pt_round_trip(tmp_path):
    P, C = 40, 16
    feats = torch.randn(P, C)
    mask = torch.rand(P) > 0.4
    p = str(tmp_path / "out" / "0.pt")
    io.save_fused_features(p, feats[mask], mask)
    blob = torch.load(p)
    assert set(blob) == {"feat", "mask_full"} and blob["feat"].dtype == torch.float16 and blob["mask_full"].dtype == torch.bool
    feat, m2 = io.load_fused_features(p, num_gaussians=P)
    assert torch.equal(m2, mask) and torch.equal(feat, feats[mask].half())
    full = io.scatter_fused_features(feat, m2, device="cpu")
    assert full.shape == (P, C) and torch.all(full[~mask] == 0) and torch.equal(full[mask], feats[mask].half().float())
    with pytest.raises(ValueError):
        io.load_fused_features(p, num_gaussians=P + 1)
    with pytest.raises(ValueError):
        io.save_fused_features(p, feats, mask)


def test_dynamic_npz(tmp_path):
    rng = np.random.default_rng(0)
    n, T = 12, 3
    np.savez(tmp_path / "params.npz", means3D=rng.standard_normal((T, n, 3)), rgb_colors=rng.random((T, n, 3)),
             unnorm_rotations=rng.standard_normal((T, n, 4)), logit_opacities=rng.standard_normal((n, 1)),
             log_scales=rng.standard_normal((n, 3)), seg_colors=rng.random((n, 3)))
    m = GaussianModel(3)
    m.load_dynamic_npz(str(tmp_path / "params.npz"), 2, device="cpu")
    z = np.load(tmp_path / "params.npz")
    assert np.allclose(m._xyz.numpy(), z["means3D"][2].astype(np.float32))
    assert m._features_dc.shape == (n, 1, 3) and m._features_rest.shape == (n, 15, 3)
    assert np.allclose(m._features_dc[:, 0].numpy(), (z["rgb_colors"][2].astype(np.float32) - 0.5) / io.C0, atol=1e-6)
    assert m.is_fg.shape == (n,)
