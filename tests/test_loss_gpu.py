"""GPU: the fused L1 + D-SSIM loss (csrc/loss.cu via loss_utils.py) against torch float64 autograd of the
reference's expressions (utils/loss_utils.py, train.py:141-149), its autograd behaviour, and one training step
and a short fit through the rasterizer."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from loss_ref import photometric_torch, ssim_torch, window  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


def _view(c):
    return SimpleNamespace(image_width=c.image_width, image_height=c.image_height, FoVx=c.FoVx, FoVy=c.FoVy,
                           world_view_transform=torch.as_tensor(c.world_view_transform, device=DEV),
                           full_proj_transform=torch.as_tensor(c.full_proj_transform, device=DEV),
                           camera_center=torch.as_tensor(c.camera_center, device=DEV))


def _model(scene, device=DEV):
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    return GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs,
                                        device=device)


def _uniform_pair(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.rand(shape, generator=g, device=DEV), torch.rand(shape, generator=g, device=DEV))


def _rendered_pair(H, W, P=30000, seed=4):
    """A target rendered from a synthetic scene and a 'rendering' of a perturbed copy of it, both (3,H,W)."""
    from semantic_gaussians_b200.renderer import render
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    scene = make_scene(P, seed=seed, sh=True, scale_mean=0.04)
    rng = np.random.default_rng(seed)
    v = _view(orbit_cameras(1, W, H)[0])
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        gt = render(v, _model(scene), Pipe, bg)["render"].clone()
        scene.xyz = (scene.xyz + rng.normal(0, 0.01, scene.xyz.shape)).astype(np.float32)
        img = render(v, _model(scene), Pipe, bg)["render"].clone()
    return img, gt


def _three_ways(x, y, fn_ours, fn_torch):
    """(value, grad) of ours, of the fp32 torch expressions and of float64 torch on the same fp32 window taps."""
    xo = x.clone().requires_grad_(True)
    vo = fn_ours(xo, y)
    vo.backward()
    x32 = x.clone().requires_grad_(True)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the fp32 yardstick is true fp32, not TF32 convolutions
    try:
        v32 = fn_torch(x32, y, window(torch.float32, DEV))
        v32.backward()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    x64 = x.double().requires_grad_(True)
    v64 = fn_torch(x64, y.double(), window(torch.float64, DEV, separable_fp64=True))
    v64.backward()
    return ((float(vo.detach()), xo.grad.double()), (float(v32.detach()), x32.grad.double()),
            (float(v64.detach()), x64.grad))


def _assert_no_less_accurate(ours, t32, t64, what):
    (vo, go), (v32, g32), (v64, g64) = ours, t32, t64
    e_ours, e32 = abs(vo - v64), abs(v32 - v64)
    assert e_ours <= 2 * e32 + 1e-6, f"{what}: loss error {e_ours:.3g} vs fp32 torch {e32:.3g}"
    ge_ours = float((go - g64).abs().max())
    ge32 = float((g32 - g64).abs().max())
    gmax = float(g64.abs().max())
    assert ge_ours <= 2 * ge32 + 1e-4 * gmax, f"{what}: grad error {ge_ours:.3g} vs fp32 torch {ge32:.3g} (max {gmax:.3g})"


CASES = [((3, 1080, 1920), False), ((3, 968, 1296), True), ((3, 37, 53), False), ((1, 5, 7), False),
         ((2, 3, 64, 80), False)]


@pytest.mark.parametrize("shape,cut_edge", CASES)
def test_photometric_loss_parity_uniform(shape, cut_edge):
    from semantic_gaussians_b200.loss_utils import photometric_loss
    x, y = _uniform_pair(shape, seed=len(shape) + shape[-1])
    res = _three_ways(x, y, lambda a, b: photometric_loss(a, b, 0.2, cut_edge)[0],
                      lambda a, b, w: photometric_torch(a, b, w, 0.2, cut_edge)[0])
    _assert_no_less_accurate(*res, what=f"photometric {shape}")
    # the detached L1 term train.py logs
    _, l1 = photometric_loss(x, y, 0.2, cut_edge)
    _, l1_64 = photometric_torch(x.double(), y.double(), window(torch.float64, DEV), 0.2, cut_edge)
    assert not l1.requires_grad and abs(float(l1) - float(l1_64)) <= 1e-6 * float(l1_64) + 1e-7


@pytest.mark.parametrize("shape,cut_edge", [c for c in CASES if c[0][0] == 3 and len(c[0]) == 3])
def test_photometric_loss_parity_rendered(shape, cut_edge):
    from semantic_gaussians_b200.loss_utils import photometric_loss
    x, y = _rendered_pair(*shape[1:])
    res = _three_ways(x, y, lambda a, b: photometric_loss(a, b, 0.2, cut_edge)[0],
                      lambda a, b, w: photometric_torch(a, b, w, 0.2, cut_edge)[0])
    _assert_no_less_accurate(*res, what=f"photometric rendered {shape}")


@pytest.mark.parametrize("shape", [(3, 1080, 1920), (3, 37, 53), (1, 5, 7), (2, 3, 64, 80)])
def test_ssim_parity(shape):
    from semantic_gaussians_b200.loss_utils import ssim
    x, y = _uniform_pair(shape, seed=7)
    y = (0.7 * x + 0.3 * y).contiguous()      # correlated, so SSIM is far from 0
    res = _three_ways(x, y, ssim, ssim_torch)
    _assert_no_less_accurate(*res, what=f"ssim {shape}")


def test_gradient_scales_with_the_upstream_gradient():
    from semantic_gaussians_b200.loss_utils import photometric_loss, ssim
    x, y = _uniform_pair((3, 90, 120), seed=11)
    a = x.clone().requires_grad_(True)
    ssim(a, y).backward()
    b = x.clone().requires_grad_(True)
    (0.2 * (1 - ssim(b, y))).backward()
    # fp32 rounding of the scaled weights, relative to the largest entry (the L1 and SSIM terms cancel in places)
    torch.testing.assert_close(b.grad, -0.2 * a.grad, rtol=0, atol=1e-6 * float(a.grad.abs().max()) * 0.2)
    c = x.clone().requires_grad_(True)
    photometric_loss(c, y)[0].backward()
    d = x.clone().requires_grad_(True)
    (3.7 * photometric_loss(d, y)[0]).backward()
    torch.testing.assert_close(d.grad, 3.7 * c.grad, rtol=0, atol=1e-6 * float(c.grad.abs().max()) * 3.7)


def test_gradient_is_zero_outside_the_crop():
    from semantic_gaussians_b200.loss_utils import photometric_loss
    x, y = _uniform_pair((3, 250, 430), seed=12)
    x.requires_grad_(True)
    photometric_loss(x, y, cut_edge=True)[0].backward()
    g = x.grad
    assert g.shape == x.shape
    ch, cw = 2, 4
    inner = torch.zeros_like(g, dtype=torch.bool)
    inner[:, ch:-ch, cw:-cw] = True
    assert not g[~inner].any()
    assert bool((g[inner] != 0).float().mean() > 0.99)


def test_non_contiguous_inputs_give_the_same_answers():
    from semantic_gaussians_b200.loss_utils import photometric_loss, ssim
    x, y = _uniform_pair((3, 130, 170), seed=13)

    def run(a, b, cut):
        a = a.detach().requires_grad_(True)
        loss, l1 = photometric_loss(a, b, 0.2, cut)
        loss.backward()
        return loss.detach(), l1, a.grad

    for cut in (False, True):
        want = run(x, y, cut)
        cl = lambda t: t.permute(1, 2, 0).contiguous().permute(2, 0, 1)          # channels-last views
        big = torch.zeros(3, 150, 200, device=DEV)
        big[:, 7:137, 11:181] = x
        for a, b in ((cl(x), cl(y)), (cl(x), y), (big[:, 7:137, 11:181], y)):
            got = run(a, b, cut)
            torch.testing.assert_close(got[0], want[0], rtol=1e-6, atol=0)
            torch.testing.assert_close(got[1], want[1], rtol=1e-6, atol=0)
            assert torch.equal(got[2], want[2])
    # (N,C,H,W) whose planes do not share one stride
    x4, y4 = _uniform_pair((3, 2, 40, 50), seed=14)
    xt, yt = x4.transpose(0, 1), y4.transpose(0, 1)
    a = xt.detach().requires_grad_(True)
    s = ssim(a, yt)
    s.backward()
    b = xt.contiguous().requires_grad_(True)
    s2 = ssim(b, yt.contiguous())
    s2.backward()
    torch.testing.assert_close(s, s2, rtol=1e-6, atol=0)
    assert torch.equal(a.grad, b.grad)


def test_two_calls_give_bit_identical_gradients():
    from semantic_gaussians_b200.loss_utils import photometric_loss
    x, y = _uniform_pair((3, 968, 1296), seed=15)
    grads = []
    for _ in range(2):
        a = x.clone().requires_grad_(True)
        photometric_loss(a, y, 0.2, True)[0].backward()
        grads.append(a.grad)
    assert torch.equal(grads[0], grads[1])


def test_forward_and_backward_never_synchronise():
    from semantic_gaussians_b200.loss_utils import photometric_loss, ssim
    x, y = _uniform_pair((3, 200, 300), seed=16)
    a = x.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss, l1 = photometric_loss(a, y, 0.2, True)
        loss.backward()
        s = ssim(a, y)
        (1 - s).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(a.grad).all() and float(l1) > 0


def test_training_step_through_the_rasterizer_matches_torch_loss():
    """render -> loss -> backward at 320x240: the Gaussian parameter gradients with the fused loss equal those
    with the reference's torch expressions."""
    from semantic_gaussians_b200.renderer import render
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    scene = make_scene(20000, seed=31, sh=True, scale_mean=0.04)
    v = _view(orbit_cameras(3, 320, 240)[1])
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        gt = render(v, _model(scene), Pipe, bg)["render"].clone()
    rng = np.random.default_rng(2)
    scene.xyz = (scene.xyz + rng.normal(0, 0.01, scene.xyz.shape)).astype(np.float32)
    scene.opacity = np.clip(scene.opacity * rng.uniform(0.8, 1.2, scene.opacity.shape), 0.01, 0.99).astype(np.float32)
    names = ("_xyz", "_opacity", "_scaling", "_rotation", "_features_dc", "_features_rest")

    def step(loss_fn):
        m = _model(scene)
        for n in names:
            getattr(m, n).requires_grad_(True)
        img = render(v, m, Pipe, bg)["render"]
        loss_fn(img, gt).backward()
        return {n: getattr(m, n).grad.clone() for n in names}

    from semantic_gaussians_b200.loss_utils import photometric_loss
    ours = step(lambda a, b: photometric_loss(a, b, 0.2, True)[0])
    ref = step(lambda a, b: photometric_torch(a, b, window(torch.float32, DEV), 0.2, True)[0])
    for n in names:
        scale = float(ref[n].abs().max())
        assert scale > 0, n
        err = float((ours[n] - ref[n]).abs().max())
        assert err <= 1e-4 * scale, f"{n}: {err:.3g} vs max {scale:.3g}"


def test_short_rgb_fit_with_l1_dssim_and_cut_edge():
    """test_train_loop_gpu.py's fit with train.py's full loss: lambda_dssim = 0.2 and the border crop."""
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.loss_utils import photometric_loss
    from semantic_gaussians_b200.renderer import render
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    torch.manual_seed(0)
    scene = make_scene(4000, seed=21, sh=True, scale_mean=0.05)
    gt = _model(scene)
    views = [_view(c) for c in orbit_cameras(6, 160, 120)]
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        targets = [render(v, gt, Pipe, bg)["render"].clone() for v in views]
    rng = np.random.default_rng(0)
    keep = rng.choice(4000, 1500, replace=False)
    pts = scene.xyz[keep] + rng.normal(0, 0.01, (1500, 3)).astype(np.float32)
    m = GaussianModel(3).create_from_pcd(pts, rng.uniform(0.3, 0.7, (1500, 3)), spatial_lr_scale=1.0, device=DEV)
    m.active_sh_degree = 0
    args = SimpleNamespace(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                           position_lr_max_steps=300, feature_lr=2.5e-3, opacity_lr=0.05, scaling_lr=5e-3, rotation_lr=1e-3)
    m.training_setup(args)
    losses, l1s = [], []
    for it in range(1, 241):
        m.update_learning_rate(it)
        v = views[it % len(views)]
        out = render(v, m, Pipe, bg)
        loss, l1 = photometric_loss(out["render"], targets[it % len(views)], 0.2, cut_edge=True)
        loss.backward()
        losses.append(loss.detach())
        l1s.append(l1)
        with torch.no_grad():
            vis, radii = out["visibility_filter"], out["radii"]
            m.max_radii2D[vis] = torch.max(m.max_radii2D[vis], radii[vis].float())
            m.add_densification_stats(out["viewspace_points"], vis)
            if it % 60 == 0:
                m.densify_and_prune(0.0002, 0.005, 3.0, None)
            m.optimizer.step()
            m.optimizer.zero_grad(set_to_none=True)
    losses = torch.stack(losses).cpu().numpy()
    l1s = torch.stack(l1s).cpu().numpy()
    first, last = float(np.mean(losses[:10])), float(np.mean(losses[-10:]))
    print(f"fit: loss first10 {first:.4f} last10 {last:.4f} ratio {last / first:.3f}; "
          f"l1 {np.mean(l1s[:10]):.4f} -> {np.mean(l1s[-10:]):.4f}")
    assert np.isfinite(losses).all() and np.isfinite(l1s).all()
    assert last < 0.8 * first, (first, last)
