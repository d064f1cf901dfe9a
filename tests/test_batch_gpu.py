"""Batched multi-view path (BASELINE config K4): render_chn_batch / render_batch over
sgb_forward_geometry_batch / sgb_forward_render_batch / sgb_backward_batch must give, per view, exactly what the
single-view calls give, and gradients equal to the sum over the views (fp32 re-association only: the (P, C)
feature gradient is accumulated in place across the views by red.add)."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from util import frac_bad, rel_err  # noqa: E402

from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.renderer import render, render_batch, render_chn, render_chn_batch  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


class Cam:
    pass


def _cams(n, W, H, dev):
    out = []
    for c in orbit_cameras(n, W, H):
        v = Cam()
        v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
        v.world_view_transform = torch.as_tensor(c.world_view_transform, device=dev)
        v.full_proj_transform = torch.as_tensor(c.full_proj_transform, device=dev)
        v.camera_center = torch.as_tensor(c.camera_center, device=dev)
        out.append(v)
    return out


def _model(P, C, dev, sh=False, seed=5):
    scene = make_scene(P, seed=seed, channels=C, sh=sh, scale_mean=0.03)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, scene.shs, device=dev)
    feats = torch.as_tensor(scene.features, device=dev).contiguous().requires_grad_(True) if C else None
    leaves = [pc._xyz, pc._scaling, pc._rotation, pc._opacity]
    if sh:
        leaves += [pc._features_dc, pc._features_rest]
    for t in leaves:
        t.requires_grad_(True)
    return pc, feats, leaves


def _grads(leaves, feats):
    out = [t.grad.clone() for t in leaves]
    if feats is not None:
        out.append(feats.grad.clone())
    for t in leaves + ([feats] if feats is not None else []):
        t.grad = None
    return out


@pytest.mark.parametrize("C,V", [(32, 3), (100, 5), (256, 11)])   # 11 > SGB_MAX_BATCH: the wrapper splits the batch
def test_render_chn_batch_equals_per_view_calls(C, V):
    dev = torch.device("cuda:0")
    W, H = 320, 240
    pc, feats, leaves = _model(30000, C, dev)
    cams = _cams(V, W, H, dev)
    bg = torch.linspace(0.0, 0.3, C, device=dev)
    g = torch.Generator(device=dev).manual_seed(1)
    dLs = [torch.randn((C, H, W), device=dev, generator=g) for _ in range(V)]

    single = [render_chn(c, pc, Pipe, bg, num_channels=C, override_color=feats) for c in cams]
    sum((o["render"] * d).sum() for o, d in zip(single, dLs)).backward()
    g_single = _grads(leaves, feats)
    vs_single = [o["viewspace_points"].grad.clone() for o in single]

    batch = render_chn_batch(cams, pc, Pipe, bg, num_channels=C, override_color=feats)
    assert len(batch) == V
    for o, b in zip(single, batch):
        assert torch.equal(o["radii"], b["radii"])
        assert torch.equal(o["render"].detach().view(torch.int32), b["render"].detach().view(torch.int32))
        assert torch.equal(o["visibility_filter"], b["visibility_filter"])
    sum((o["render"] * d).sum() for o, d in zip(batch, dLs)).backward()
    g_batch = _grads(leaves, feats)
    for a, b in zip(g_single, g_batch):
        # both sides sum fp32 partial gradients with red.global in scheduling order: 1e-4 relative + 1e-4 of the scale
        assert frac_bad(b, a, rtol=1e-4, atol_scale=1e-4) == 0.0
        assert rel_err(b, a) < 1e-4
    for o, want in zip(batch, vs_single):        # per-view screen-space gradients (densification statistics)
        assert frac_bad(o["viewspace_points"].grad, want, rtol=1e-4, atol_scale=1e-4) == 0.0


def test_render_batch_rgbd_sh_path_equals_per_view_calls():
    """C = 3 with spherical harmonics: every view keeps its own RGB gradient (it feeds that view's SH backward)."""
    dev = torch.device("cuda:0")
    W, H, V = 256, 192, 4
    pc, _, leaves = _model(20000, 0, dev, sh=True)
    cams = _cams(V, W, H, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    g = torch.Generator(device=dev).manual_seed(2)
    dLs = [torch.randn((3, H, W), device=dev, generator=g) for _ in range(V)]
    single = [render(c, pc, Pipe, bg) for c in cams]
    sum((o["render"] * d).sum() for o, d in zip(single, dLs)).backward()
    g_single = _grads(leaves, None)
    batch = render_batch(cams, pc, Pipe, bg)
    for o, b in zip(single, batch):
        assert torch.equal(o["render"].detach().view(torch.int32), b["render"].detach().view(torch.int32))
        assert torch.equal(o["depth"].view(torch.int32), b["depth"].view(torch.int32))
        assert torch.equal(o["radii"], b["radii"])
    sum((o["render"] * d).sum() for o, d in zip(batch, dLs)).backward()
    g_batch = _grads(leaves, None)
    for a, b in zip(g_single, g_batch):
        assert frac_bad(b, a, rtol=1e-4, atol_scale=1e-4) == 0.0


def test_forward_forward_backward_backward_reuses_every_views_weight_rows():
    """Several single-view forwards followed by their backwards (what autograd does for a loss summed over views):
    every view's backward must see ITS weight rows (per-ctx pool slots), not the last forward's."""
    dev = torch.device("cuda:0")
    C, W, H, V = 64, 320, 240, 4
    pc, feats, leaves = _model(30000, C, dev, seed=9)
    cams = _cams(V, W, H, dev)
    bg = torch.zeros(C, device=dev)
    g = torch.Generator(device=dev).manual_seed(3)
    dLs = [torch.randn((C, H, W), device=dev, generator=g) for _ in range(V)]
    # reference: strictly interleaved forward / backward per view
    want = None
    for c, d in zip(cams, dLs):
        render_chn(c, pc, Pipe, bg, num_channels=C, override_color=feats)["render"].backward(d)
    want = _grads(leaves, feats)
    outs = [render_chn(c, pc, Pipe, bg, num_channels=C, override_color=feats) for c in cams]
    for o, d in zip(reversed(outs), reversed(dLs)):
        o["render"].backward(d)
    got = _grads(leaves, feats)
    for a, b in zip(want, got):
        assert frac_bad(b, a, rtol=1e-4, atol_scale=1e-4) == 0.0


def test_batch_argument_validation():
    from semantic_gaussians_b200 import channel_rasterization as chn
    dev = torch.device("cuda:0")
    pc, feats, _ = _model(1000, 8, dev)
    cams = _cams(2, 64, 48, dev)
    mk = lambda cam, bg, H: chn.GaussianRasterizationSettings(
        H, 64, math.tan(cam.FoVx / 2), math.tan(cam.FoVy / 2), bg, 1.0, cam.world_view_transform,
        cam.full_proj_transform, 0, cam.camera_center, False, False, 8)
    bg = torch.zeros(8, device=dev)
    pts = [torch.zeros_like(pc.get_xyz) for _ in range(2)]
    with pytest.raises(ValueError, match="must share"):
        chn.GaussianRasterizer.rasterize_batch(pc.get_xyz, pts, pc.get_opacity, [mk(cams[0], bg, 48), mk(cams[1], bg, 32)],
                                               colors_precomp=feats, scales=pc.get_scaling, rotations=pc.get_rotation)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        chn.GaussianRasterizer.rasterize_batch(pc.get_xyz, pts, pc.get_opacity, [mk(cams[0], bg, 48), mk(cams[1], bg, 48)],
                                               scales=pc.get_scaling, rotations=pc.get_rotation)
