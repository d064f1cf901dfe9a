"""Colour and a feature table through one geometry pass and one binning per view (render_with_features /
render_with_features_batch, sgb_forward_render_joint_batch / sgb_backward_joint_batch):

  * forward: RGB, median depth, radii, final_T and n_contrib bitwise render()'s, expected depth / alpha bitwise
    render_with_depth()'s, the feature image bitwise render_chn()'s with the same table and background;
  * backward: every gradient is the sum of the separate render_with_depth() and render_chn() backwards (1e-4);
  * batches equal per-view calls (split past the native limit), no host synchronisation in the backward, and a short
    joint fit with densification keeps the feature table row-aligned while the loss falls."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from raster_check import read_state  # noqa: E402
from util import frac_bad  # noqa: E402

from semantic_gaussians_b200 import _lib, rasterizer  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.renderer import (_prepare, render, render_chn, render_with_depth,  # noqa: E402
                                              render_with_features, render_with_features_batch)
from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


class CovPipe(Pipe):
    compute_cov3d_python = True


class PySHPipe(Pipe):
    convert_shs_python = True


class Cam:
    pass


def _cam(c):
    v = Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
    v.world_view_transform = torch.as_tensor(c.world_view_transform, device=DEV)
    v.full_proj_transform = torch.as_tensor(c.full_proj_transform, device=DEV)
    v.camera_center = torch.as_tensor(c.camera_center, device=DEV)
    return v


def _model(P, sh_degree=3, seed=7, scale_mean=0.03):
    scene = make_scene(P, seed=seed, sh=True, scale_mean=scale_mean)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, scene.shs, device=DEV)
    pc.active_sh_degree = sh_degree
    leaves = [pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest]
    for t in leaves:
        t.requires_grad_(True)
    return pc, leaves


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _features(P, c, seed=5):
    return torch.randn((P, c), device=DEV, generator=_gen(seed)).requires_grad_(True)


def _take_grads(ts):
    out = [torch.zeros_like(t) if t.grad is None else t.grad.clone() for t in ts]
    for t in ts:
        t.grad = None
    return out


BG = lambda: torch.tensor([0.2, 0.4, 0.6], device=DEV)


def _bg_features(c):
    return torch.linspace(-0.5, 0.5, c, device=DEV)


def _equal(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(a, b), float((a.float() - b.float()).abs().max())


# ---- forward parity --------------------------------------------------------------------------------------------
FWD = {  # name: (P, W, H, sh degree, pipe, override colour, camera)
    "sh3": (20000, 173, 109, 3, Pipe, False, "orbit"),
    "sh0": (20000, 173, 109, 0, Pipe, False, "orbit"),
    "override_color": (20000, 173, 109, 3, Pipe, True, "orbit"),
    "cov3d_python": (20000, 173, 109, 3, CovPipe, False, "orbit"),
    "convert_shs_python": (20000, 173, 109, 3, PySHPipe, False, "orbit"),
    "no_instances": (20000, 173, 109, 3, Pipe, False, "away"),
}


def _fwd_setup(name, c):
    P, W, H, deg, pipe, override, where = FWD[name]
    pc, _ = _model(P, deg)
    cam = orbit_cameras(4, W, H)[1] if where == "orbit" else look_at_camera((3.0, 0.0, 0.4), (6.0, 0.0, 0.4), W, H)
    colors = torch.rand((P, 3), device=DEV, generator=_gen(3)) if override else None
    return pc, _cam(cam), pipe, colors, _features(P, c), _bg_features(c)


@pytest.mark.parametrize("c", [1, 3, 4, 5, 16, 64, 256, 512])
@pytest.mark.parametrize("name", ["sh3", "sh0"])
def test_forward_is_render_render_with_depth_and_render_chn(name, c):
    pc, cam, pipe, colors, feats, bgf = _fwd_setup(name, c)
    with torch.no_grad():
        joint = render_with_features(cam, pc, pipe, BG(), feats, bgf, override_color=colors, differentiable_depth=True)
        plain = render_with_features(cam, pc, pipe, BG(), feats, bgf, override_color=colors)
        rgb = render(cam, pc, pipe, BG(), override_color=colors)
        rgbd = render_with_depth(cam, pc, pipe, BG(), override_color=colors)
        chn = render_chn(cam, pc, pipe, bgf, num_channels=c, override_color=feats)
    assert int((rgb["radii"] > 0).sum()) > 1000
    for out in (joint, plain):
        for k in ("render", "depth", "radii", "visibility_filter"):
            _equal(out[k], rgb[k])
        _equal(out["features"], chn["render"])
    _equal(joint["expected_depth"], rgbd["expected_depth"])
    _equal(joint["alpha"], rgbd["alpha"])
    assert "expected_depth" not in plain


@pytest.mark.parametrize("name", ["override_color", "cov3d_python", "convert_shs_python", "no_instances"])
@pytest.mark.parametrize("c", [4, 64])
def test_forward_options(name, c):
    pc, cam, pipe, colors, feats, bgf = _fwd_setup(name, c)
    with torch.no_grad():
        joint = render_with_features(cam, pc, pipe, BG(), feats, bgf, override_color=colors, differentiable_depth=True)
        rgbd = render_with_depth(cam, pc, pipe, BG(), override_color=colors)
        chn = render_chn(cam, pc, pipe, bgf, num_channels=c, override_color=feats)
    for k in ("render", "depth", "radii", "expected_depth", "alpha"):
        _equal(joint[k], rgbd[k])
    _equal(joint["features"], chn["render"])
    if name == "no_instances":
        assert int(joint["radii"].max()) == 0
        _equal(joint["features"], bgf[:, None, None].expand_as(joint["features"]).contiguous())


@pytest.mark.parametrize("c", [3, 64])
def test_forward_state_is_renders(c):
    """Instance count, radii, final_T and n_contrib of the joint forward are the RGB forward's."""
    pc, cam, pipe, _, feats, bgf = _fwd_setup("sh3", c)
    pts, common, call = _prepare(cam, pc, pipe, 1.0, None, None, None, None)
    cams = [(common["viewmatrix"], common["projmatrix"], common["campos"], common["tanfovx"], common["tanfovy"])]
    args = (cams, BG(), call["means3D"], None, call["opacities"], call["scales"], call["rotations"], 1.0, None,
            common["image_height"], common["image_width"], call["shs"], common["sh_degree"], False, False)
    with torch.no_grad():
        _, (R0, _, radii0, geom0, bin0, img0, *_) = rasterizer._forward(True, "rgb", *args[:-1], False, 3)
        _, (R1, _, radii1, geom1, bin1, img1, *_), _, _ = rasterizer._forward_joint("joint", *args, feats, bgf)
    assert R0 == R1
    _equal(radii0[0], radii1[0])
    P, W, H = call["means3D"].shape[0], common["image_width"], common["image_height"]
    s0 = read_state(_lib.load(), P, R0[0], W, H, geom0[0], bin0[0], img0[0])
    s1 = read_state(_lib.load(), P, R1[0], W, H, geom1[0], bin1[0], img1[0])
    for k in ("final_T", "n_contrib", "point_list", "ranges"):
        _equal(s0[k], s1[k])
    vis = radii0[0] > 0  # preprocess writes the records of the Gaussians it keeps only
    for k in ("means2D", "conic_opacity"):
        _equal(s0[k][vis], s1[k][vis])


def test_empty_scene():
    pc, _ = _model(10)
    for t in (pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest):
        t.data = t.data[:0]
    cam = _cam(orbit_cameras(1, 67, 45)[0])
    feats = torch.zeros((0, 8), device=DEV, requires_grad=True)
    out = render_with_features(cam, pc, Pipe, BG(), feats, _bg_features(8), differentiable_depth=True)
    assert out["render"].shape == (3, 45, 67) and out["features"].shape == (8, 45, 67)
    assert float(out["render"].abs().max()) == 0.0 and float(out["features"].abs().max()) == 0.0
    (out["render"].sum() + out["features"].sum()).backward()
    assert feats.grad.shape == (0, 8)


@pytest.mark.parametrize("V", [1, 3, 9])
@pytest.mark.parametrize("c", [4, 64])
def test_batch_equals_per_view_calls(V, c):
    W, H = 131, 97
    pc, leaves = _model(20000)
    cams = [_cam(x) for x in orbit_cameras(V, W, H)]
    feats, bgf = _features(20000, c), _bg_features(c)
    batch = render_with_features_batch(cams, pc, Pipe, BG(), feats, bgf, differentiable_depth=True)
    assert len(batch) == V
    a = [torch.rand((3, H, W), device=DEV, generator=_gen(10 + v)) for v in range(V)]
    b = [torch.rand((c, H, W), device=DEV, generator=_gen(40 + v)) for v in range(V)]
    loss = lambda outs: sum((o["render"] * x).sum() + (o["features"] * y).sum() + o["expected_depth"].sum()
                            for o, x, y in zip(outs, a, b))
    loss(batch).backward()
    g_batch = _take_grads(leaves + [feats])
    single = [render_with_features(cam, pc, Pipe, BG(), feats, bgf, differentiable_depth=True) for cam in cams]
    for o, s in zip(batch, single):
        for k in ("render", "depth", "radii", "features", "expected_depth", "alpha"):
            _equal(o[k], s[k])
    loss(single).backward()
    for x, y in zip(_take_grads(leaves + [feats]), g_batch):
        assert frac_bad(x, y, rtol=1e-4, atol_scale=1e-4) == 0.0
    for o, s in zip(batch, single):
        assert frac_bad(o["viewspace_points"].grad, s["viewspace_points"].grad, rtol=1e-4, atol_scale=1e-4) == 0.0


# ---- backward parity -------------------------------------------------------------------------------------------
BWD = {  # name: (sh degree, pipe, override colour, c, depth terms)
    "sh3_c16": (3, Pipe, False, 16, True),
    "sh3_c64": (3, Pipe, False, 64, True),
    "sh0_c3": (0, Pipe, False, 3, True),
    "sh3_c512": (3, Pipe, False, 512, False),
    "override_c5": (3, Pipe, True, 5, True),
    "cov3d_c64": (3, CovPipe, False, 64, True),
    "cov3d_c1": (3, CovPipe, False, 1, False),
}


@pytest.mark.parametrize("name", list(BWD))
def test_backward_is_the_sum_of_the_separate_backwards(name):
    deg, pipe, override, c, depth_terms = BWD[name]
    P, W, H = 20000, 157, 103
    pc, leaves = _model(P, deg)
    cam = _cam(orbit_cameras(4, W, H)[2])
    colors = torch.rand((P, 3), device=DEV, generator=_gen(3)).requires_grad_(True) if override else None
    feats, bgf = _features(P, c), _bg_features(c)
    ts = leaves + [feats] + ([colors] if override else [])
    a = torch.randn((3, H, W), device=DEV, generator=_gen(11))
    b = torch.randn((2, H, W), device=DEV, generator=_gen(12)) * 0.1
    f = torch.randn((c, H, W), device=DEV, generator=_gen(13))
    out = render_with_features(cam, pc, pipe, BG(), feats, bgf, override_color=colors,
                               differentiable_depth=depth_terms)
    loss = (out["render"] * a).sum() + (out["features"] * f).sum()
    if depth_terms:
        loss = loss + (out["expected_depth"] * b[0]).sum() + (out["alpha"] * b[1]).sum()
    loss.backward()
    g_joint, vs_joint = _take_grads(ts), out["viewspace_points"].grad
    sep = (render_with_depth if depth_terms else render)(cam, pc, pipe, BG(), override_color=colors)
    chn = render_chn(cam, pc, pipe, bgf, num_channels=c, override_color=feats)
    loss = (sep["render"] * a).sum() + (chn["render"] * f).sum()
    if depth_terms:
        loss = loss + (sep["expected_depth"] * b[0]).sum() + (sep["alpha"] * b[1]).sum()
    loss.backward()
    g_sep = _take_grads(ts)
    vs_sep = sep["viewspace_points"].grad + chn["viewspace_points"].grad
    assert float(g_sep[6].abs().max()) > 0.0 and float(g_sep[0].abs().max()) > 0.0
    for i, (x, y) in enumerate(zip(g_joint, g_sep)):
        assert frac_bad(x, y, rtol=1e-4, atol_scale=1e-4) == 0.0, (i, float((x - y).abs().max()))
    assert frac_bad(vs_joint, vs_sep, rtol=1e-4, atol_scale=1e-4) == 0.0


def test_loss_on_one_image_only():
    """A loss on the feature image alone gives render_chn's gradients; on the RGB image alone render()'s."""
    P, W, H, c = 20000, 128, 96, 32
    pc, leaves = _model(P)
    cam = _cam(orbit_cameras(4, W, H)[0])
    feats, bgf = _features(P, c), _bg_features(c)
    ts = leaves + [feats]
    render_with_features(cam, pc, Pipe, BG(), feats, bgf)["features"].square().sum().backward()
    g_joint = _take_grads(ts)
    render_chn(cam, pc, Pipe, bgf, num_channels=c, override_color=feats)["render"].square().sum().backward()
    for x, y in zip(g_joint, _take_grads(ts)):
        assert frac_bad(x, y, rtol=1e-4, atol_scale=1e-4) == 0.0
    render_with_features(cam, pc, Pipe, BG(), feats, bgf)["render"].square().sum().backward()
    g_joint = _take_grads(ts)
    render(cam, pc, Pipe, BG())["render"].square().sum().backward()
    g_rgb = _take_grads(ts)
    for x, y in zip(g_joint, g_rgb):
        assert frac_bad(x, y, rtol=1e-4, atol_scale=1e-4) == 0.0
    assert float(g_joint[-1].abs().max()) == 0.0


def test_backward_adds_no_host_synchronisation():
    pc, leaves = _model(20000)
    cam = _cam(orbit_cameras(4, 160, 96)[1])
    feats, bgf = _features(20000, 64), _bg_features(64)
    for warm in (True, False):
        out = render_with_features(cam, pc, Pipe, BG(), feats, bgf, differentiable_depth=True)
        loss = out["render"].sum() + out["features"].sum() + out["expected_depth"].sum()
        torch.cuda.synchronize()
        if not warm:
            torch.cuda._sleep(2_000_000_000)
        loss.backward()
        done = torch.cuda.Event()
        done.record()
        if not warm:
            assert not done.query(), "the backward waited for the GPU"
        torch.cuda.synchronize()
    assert float(feats.grad.abs().max()) > 0.0


# ---- a joint training loop with densification ---------------------------------------------------------------
def test_joint_fit_with_densification():
    """Fit colours and a c = 16 field decoded to 64 channels against a target scene, with densification every 20
    steps (the Gaussians in the top 3 % of the screen-space gradient statistic): the row counts stay consistent, and
    the decoded feature loss and the photometric loss fall.  A last step runs under torch's sync debug mode, which sees
    synchronisations made through torch only: it shows that the step adds none there.  The native waits (the
    instance counts and the weight-pool check of the forward) are not visible to it; that the backward adds no wait
    is test_backward_adds_no_host_synchronisation's check."""
    from semantic_gaussians_b200.loss_utils import photometric_loss
    from semantic_gaussians_b200.semantic import decoded_feature_map_loss_and_grads
    W, H, c, Cdec, P = 160, 120, 16, 64, 8000
    cams = [_cam(x) for x in orbit_cameras(4, W, H)]
    tgt, _ = _model(P, seed=21, scale_mean=0.04)
    dec_true = torch.randn((Cdec, c), device=DEV, generator=_gen(1))
    tgt_feats = torch.randn((P, c), device=DEV, generator=_gen(2))
    with torch.no_grad():
        targets = [render_with_features(cam, tgt, Pipe, BG(), tgt_feats, torch.zeros(c, device=DEV)) for cam in cams]
        gt_feat = [torch.einsum("Cc,chw->Chw", dec_true, t["features"]).contiguous() for t in targets]
    pc, _ = _model(P, seed=21, scale_mean=0.04)
    with torch.no_grad():
        pc._xyz += 0.02 * torch.randn(pc._xyz.shape, device=DEV, generator=_gen(4))
    pc.create_semantic(c)
    pc.spatial_lr_scale = 1.0
    args = SimpleNamespace(percent_dense=0.01, position_lr_init=1e-3, position_lr_final=1e-3,
                           position_lr_delay_mult=1.0, position_lr_max_steps=1000, feature_lr=2.5e-3,
                           opacity_lr=0.05, scaling_lr=5e-3, rotation_lr=1e-3, semantic_feature_lr=5e-2,
                           optimizer_type="sparse_adam")
    pc.training_setup(args)
    decoder = torch.nn.Linear(c, Cdec, bias=False).to(DEV)
    pc.optimizer.add_param_group({"params": [decoder.weight], "lr": 1e-2, "name": "decoder"})
    bg, bgf = BG(), torch.zeros(c, device=DEV)  # made once: a host-to-device copy waits for the device
    LAMBDA = 0.1  # weight of the feature loss against the photometric loss

    def step(i, stats=True):
        cam, tg, gf = cams[i % 4], targets[i % 4], gt_feat[i % 4]
        out = render_with_features(cam, pc, Pipe, bg, pc._features_semantic, bgf)
        rgb_loss, _ = photometric_loss(out["render"], tg["render"])
        f_loss, g_r, g_w, _ = decoded_feature_map_loss_and_grads(out["features"], decoder.weight, gf, loss_type="l2")
        torch.autograd.backward([rgb_loss, out["features"]], [None, LAMBDA * g_r])
        decoder.weight.grad = LAMBDA * g_w
        vis = out["visibility_filter"]
        if stats:
            with torch.no_grad():
                pc.max_radii2D[vis] = torch.max(pc.max_radii2D[vis], out["radii"][vis].float())
                pc.add_densification_stats(out["viewspace_points"], vis)
        pc.optimizer.step(visibility=vis)
        pc.optimizer.zero_grad(set_to_none=True)
        return rgb_loss.detach(), f_loss.detach()

    def losses():
        with torch.no_grad():
            rgb, feat = 0.0, 0.0
            for cam, tg, gf in zip(cams, targets, gt_feat):
                out = render_with_features(cam, pc, Pipe, BG(), pc._features_semantic, bgf)
                rgb += float(photometric_loss(out["render"], tg["render"])[0])
                x = torch.einsum("Cc,chw->Chw", decoder.weight, out["features"])
                feat += float((x - gf).square().mean())
            return rgb, feat

    rgb0, feat0 = losses()
    sizes = [pc._xyz.shape[0]]
    for i in range(100):
        step(i)
        if i % 20 == 19:
            with torch.no_grad():
                stat = (pc.xyz_gradient_accum / pc.denom.clamp_min(1)).squeeze(1)
                thr = float(torch.quantile(stat[pc.denom.squeeze(1) > 0], 0.97))
            pc.densify_and_prune(thr, 0.005, 3.0, None)
            P_now = pc._xyz.shape[0]
            sizes.append(P_now)
            assert pc._features_semantic.shape == (P_now, c) and pc._times.shape == (P_now, 1)
            for g in pc.optimizer.param_groups:
                if g["name"] != "decoder":
                    assert g["params"][0].shape[0] == P_now
            assert pc.optimizer.param_groups[-1]["params"][0] is decoder.weight
    rgb1, feat1 = losses()
    print(f"\n[joint fit] P {sizes}; photometric {rgb0:.4f} -> {rgb1:.4f}; decoded feature {feat0:.4f} -> {feat1:.4f}")
    assert len(set(sizes)) > 1, "densification never changed the row count"
    assert rgb1 < rgb0 and feat1 < 0.5 * feat0, (rgb0, rgb1, feat0, feat1)
    # one more step (render, both losses, one backward, the optimiser; the masked densification statistics index
    # with a bool mask and so synchronise by design) under torch's sync debug mode: nothing in it synchronises through
    # torch; the forward's native reads (instance counts, weight-pool check) are its only waits
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        import warnings
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            step(0, stats=False)
        syncs = [x for x in w if "synchroniz" in str(x.message).lower()]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert not syncs, [str(x.message) for x in syncs]
