"""Fusion kernels vs golden vectors produced by the reference's own numpy code
(tests/golden/fusion_golden.npz) and vs the numpy oracle at other sizes: pixel indices and the
fp32 per-Gaussian sums are bit-exact."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_fusion_golden import fusion_inputs  # noqa: E402
from make_raster_golden import digest  # noqa: E402

from oracle import fusion_oracle as fo  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fusion_golden.npz")


@pytest.mark.parametrize("mode", ["none", "surface", "depth"])
def test_mapping_and_fused_features_match_reference_golden(mode):
    from semantic_gaussians_b200.fusion import PointCloudToImageMapper, normalize_fused
    dev = torch.device("cuda:0")
    scene, cams, feats, depths = fusion_inputs()
    gold = np.load(GOLD)
    w, h = cams[0].image_width, cams[0].image_height
    P, C = scene.P, feats[0].shape[0]
    xyz = torch.as_tensor(scene.xyz, device=dev)
    fs = torch.zeros((P, C), device=dev)
    cnt = torch.zeros(P, device=dev)
    for i, cam in enumerate(cams):
        mapper = PointCloudToImageMapper([w, h], 0.05, 4, cam.intrinsics(), device=dev)
        depth = {"none": None, "surface": "surface", "depth": depths[i]}[mode]
        m, weight = mapper.compute_mapping(cam.world_view_transform, scene.xyz, depth)
        assert m.dtype == np.int64 and np.array_equal(m, gold[f"{mode}_mapping_{i}"])
        assert weight.shape == (P,)
        nvis = mapper.accumulate(cam.world_view_transform, xyz, torch.from_numpy(feats[i]), fs, cnt, depth)
        assert int(nvis) == int(gold[f"{mode}_mapping_{i}"][:, 2].sum())
    normalize_fused(fs, cnt)
    assert np.array_equal(cnt.cpu().numpy().reshape(-1, 1), gold[f"{mode}_times"])
    assert np.array_equal(digest(fs.cpu().numpy()), gold[f"{mode}_fused.sha256"])


@pytest.mark.parametrize("C,dtype", [(512, np.float16), (33, np.float32)])
def test_accumulate_vs_oracle_large_channels(C, dtype):
    from semantic_gaussians_b200.fusion import PointCloudToImageMapper, normalize_fused
    dev = torch.device("cuda:0")
    scene, cams, _, depths = fusion_inputs(seed=2, P=40000, w=160, h=120, C=4, nviews=4)
    rng = np.random.default_rng(0)
    P = scene.P
    fs = torch.zeros((P, C), device=dev)
    cnt = torch.zeros(P, device=dev)
    fs_o, cnt_o = np.zeros((P, C), np.float32), np.zeros(P, np.float32)
    xyz = torch.as_tensor(scene.xyz, device=dev)
    for i, cam in enumerate(cams):
        fm = rng.standard_normal((C, 120, 160)).astype(dtype)
        mapper = PointCloudToImageMapper([160, 120], 0.1, 0, cam.intrinsics(), device=dev)
        mapper.accumulate(cam.world_view_transform, xyz, torch.from_numpy(fm), fs, cnt, depths[i])
        K = fo.rescale_intrinsics(cam.intrinsics(), [160, 120])
        m = fo.compute_mapping(cam.world_view_transform, scene.xyz, [160, 120], K, 0.1, 0, depths[i])
        fo.accumulate(fm, m, fs_o, cnt_o)
    normalize_fused(fs, cnt)
    fo.normalize(fs_o, cnt_o)
    assert np.array_equal(cnt.cpu().numpy(), cnt_o)
    assert np.array_equal(fs.cpu().numpy(), fs_o)


def test_fusion_edge_cases():
    from semantic_gaussians_b200.fusion import PointCloudToImageMapper
    dev = torch.device("cuda:0")
    scene, cams, feats, _ = fusion_inputs(seed=4, P=500, w=64, h=48, C=8, nviews=1)
    cam = cams[0]
    mapper = PointCloudToImageMapper([64, 48], 0.05, 0, cam.intrinsics(), device=dev)
    # a point (numerically) at the camera centre and one behind the camera
    pts = np.concatenate([scene.xyz, cam.camera_center[None], (2 * cam.camera_center)[None]]).astype(np.float32)
    m, _ = mapper.compute_mapping(cam.world_view_transform, pts, None)
    K = fo.rescale_intrinsics(cam.intrinsics(), [64, 48])
    want = fo.compute_mapping(cam.world_view_transform, pts, [64, 48], K, 0.05, 0, None)
    assert np.array_equal(m, want) and m[-1, 2] == 0
    # exact z = 0 (0/0 and x/0 -> nan / inf pixel coordinates) with an identity camera
    ident = np.eye(4, dtype=np.float32)
    pts0 = np.array([[0, 0, 0], [1, 0, 0], [0, -2, 0], [0.1, 0.1, 1.0], [0, 0, -1]], np.float32)
    m0, _ = mapper.compute_mapping(ident, pts0, None)
    want0 = fo.compute_mapping(ident, pts0, [64, 48], K, 0.05, 0, None)
    assert np.array_equal(m0, want0) and list(m0[:, 2]) == [0, 0, 0, 1, 0]
    # empty point set
    m0, _ = mapper.compute_mapping(cam.world_view_transform, np.zeros((0, 3), np.float32), None)
    assert m0.shape == (0, 3)
    with pytest.raises(ValueError):
        mapper.compute_mapping(cam.world_view_transform, scene.xyz, np.zeros((10, 10), np.float32))


def test_fuse_scene_rendered_depth_matches_host_round_trip():
    """fuse_scene(depth="render") (depth stays on the device) == the reference sequence
    render -> .cpu().numpy() -> compute_mapping (numpy oracle) -> gather/accumulate -> normalise, bit for bit."""
    from semantic_gaussians_b200.fusion import fuse_scene
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.renderer import render
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    dev = torch.device("cuda:0")
    P, C, w, h = 30000, 24, 160, 120
    scene = make_scene(P, 5, sh=True)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs, device=dev)
    cams = orbit_cameras(6, 320, 240)            # native camera size differs from img_dim -> override_shape path
    rng = np.random.default_rng(3)
    fmaps = [torch.from_numpy(rng.standard_normal((C, h, w)).astype(np.float16)).to(dev) for _ in cams]

    class Pipe:
        convert_shs_python = False
        compute_cov3d_python = False
        debug = False

    class View:
        pass

    views = []
    for c in cams:
        v = View()
        v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
        v.world_view_transform = torch.as_tensor(c.world_view_transform, device=dev)
        v.full_proj_transform = torch.as_tensor(c.full_proj_transform, device=dev)
        v.camera_center = torch.as_tensor(c.camera_center, device=dev)
        v.intrinsics = c.intrinsics()
        views.append(v)
    bg = torch.zeros(3, device=dev)
    pc.create_semantic(C)
    out = fuse_scene(pc, views, fmaps, Pipe, bg, [w, h], visibility_threshold=0.05, cut_boundary=4, depth="render", every=2)
    assert out["views"] == 3

    fs = np.zeros((P, C), np.float32)
    cnt = np.zeros(P, np.float32)
    for idx in range(0, 6, 2):
        d = render(views[idx], pc, Pipe, bg, override_shape=[w, h])["depth"].cpu().numpy()[0]      # fusion.py:110-120
        assert d.shape == (h, w) and d.dtype == np.float32
        K = fo.rescale_intrinsics(views[idx].intrinsics, [w, h])
        m = fo.compute_mapping(cams[idx].world_view_transform, scene.xyz, [w, h], K, 0.05, 4, d)
        fo.accumulate(fmaps[idx].cpu().numpy(), m, fs, cnt)
    seen = cnt > 0
    fo.normalize(fs, cnt)
    assert seen.sum() > 1000
    assert np.array_equal(out["mask"].cpu().numpy(), seen)
    assert np.array_equal(out["features"].cpu().numpy(), fs)
