"""Anti-aliasing on the GPU (preprocess_kernel<true>, geom_backward_kernel<*, true>; include/sgb200.h
sgb_view_inputs.antialiasing) through the Python paths.

  state ........... radii, tiles, instance counts, conics and depth order bitwise the flag-off values; the record's
                    opacity o h against float64 (tests/antialias_ref.py)
  renders ......... a flag-on render is bitwise the flag-off render given the record's opacities (RGB with median
                    depth, expected depth / alpha, C = 37, C = 256, joint, the lift's weight_sum)
  gradients ....... flag-on minus flag-off-at-o_eff per-Gaussian gradients against the float64 term, given the native
                    blend's upstream gradient; dL/do = h dL/d(o h)
  camera .......... rigid-motion identity, central differences along pose directions, bitwise reproducibility, and
                    no other gradient changes when camera gradients are asked for
  batch ........... a batch is bitwise its single views
  footprint ....... the reason for the feature: isolated sub-pixel Gaussians at 1x, 1/2x, 1/4x resolution"""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import antialias_ref as ar  # noqa: E402
from raster_check import DEV, read_state  # noqa: E402
from scene_recipes import push_sideways, set_view_space, view_space  # noqa: E402

from semantic_gaussians_b200 import _lib, rasterizer  # noqa: E402
from semantic_gaussians_b200.camera_opt import CameraPoseCorrection  # noqa: E402
from semantic_gaussians_b200.fusion import lift_views  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.renderer import (render, render_batch, render_chn, render_with_depth,  # noqa: E402
                                              render_with_features)
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False
    antialiasing = False


class AAPipe(Pipe):
    antialiasing = True


class Cam:
    pass


def _cam(c, grad=False):
    v = Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
    v.uid = 0
    for name in ("world_view_transform", "full_proj_transform", "camera_center", "projection_matrix"):
        setattr(v, name, torch.as_tensor(getattr(c, name), device=DEV).clone().requires_grad_(grad))
    return v


def _model(scene, grad=True, sh_degree=3):
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, scene.shs, device=DEV)
    pc.active_sh_degree = sh_degree
    leaves = [pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest]
    for t in leaves:
        t.requires_grad_(grad)
    return pc, leaves


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _native_forward(scene, c, aa, *, opac=None, C=3, colors=None, cov=None, sh=False, want_exp=False):
    t = lambda a: torch.as_tensor(a, device=DEV).contiguous()  # noqa: E731
    W, H = c.image_width, c.image_height
    cams = [(t(c.world_view_transform), t(c.full_proj_transform), t(c.camera_center), math.tan(c.FoVx * 0.5),
             math.tan(c.FoVy * 0.5))]
    o = t(scene.opacity) if opac is None else opac
    scales, rots = (None, None) if cov is not None else (t(scene.scales), t(scene.rotations))
    shs = t(scene.shs) if sh else None
    if not sh and colors is None:
        colors = torch.rand((scene.P, C), device=DEV, generator=_gen(1))
    bg = torch.linspace(0.05, 0.5, C, device=DEV)
    return rasterizer._forward(C <= 4, "t", cams, bg, t(scene.xyz), colors, o, scales, rots, 1.0, cov, H, W, shs,
                               3 if sh else 0, False, False, C, want_exp_alpha=want_exp, antialiasing=aa)


# ---------------------------------------------------------------- 1. state
def test_state_is_the_flag_off_state_but_opacity():
    scene = make_scene(200000, seed=3, sh=False, scale_mean=0.004)
    c = orbit_cameras(4, 640, 480)[1]
    push_sideways(scene, c, "xy", every=17)
    lib = _lib.load()
    P, W, H = scene.P, c.image_width, c.image_height
    st = {}
    with torch.no_grad():
        for aa in (False, True):
            native, (R, _, radii, geom, binning, img, *_) = _native_forward(scene, c, aa)
            torch.cuda.synchronize()
            s = read_state(lib, P, R[0], W, H, geom[0], binning[0], img[0], ("depths", "cov3D", "tiles_touched"))
            st[aa] = (R[0], radii[0].clone(), s)
    (R0, rad0, s0), (R1, rad1, s1) = st[False], st[True]
    assert R0 == R1 and torch.equal(rad0, rad1)
    for k in ("point_list", "ranges", "tiles_touched"):
        assert torch.equal(s0[k], s1[k]), k
    # the per-Gaussian record and cov3D of a culled Gaussian are never written (nor read): compare the visible ones
    seen = rad0 > 0
    for k in ("means2D", "depths", "cov3D"):
        assert torch.equal(s0[k][seen], s1[k][seen]), k
    assert torch.equal(s0["conic_opacity"][seen, :3], s1["conic_opacity"][seen, :3])
    vis = seen.cpu().numpy()
    cov = s0["cov3D"].double()
    tx, ty = math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5)
    a0, b, c0 = ar.screen_cov0(torch.as_tensor(scene.xyz, device=DEV).double(), cov,
                               np.asarray(c.world_view_transform).reshape(-1), W, H, tx, ty)
    r, h, active = ar.h_of(a0.cpu().numpy(), b.cpu().numpy(), c0.cpu().numpy())
    want = scene.opacity.reshape(-1).astype(np.float64) * h
    got = s1["conic_opacity"][:, 3].double().cpu().numpy()
    assert np.equal(s0["conic_opacity"][:, 3].cpu().numpy(), scene.opacity.reshape(-1))[vis].all()
    # fp32: the rounding of det C0 (a difference of products) relative to det C, and a few ulps of the product
    tol = 2e-6 * want + 1e-6 * scene.opacity.reshape(-1) * (np.abs(a0.cpu().numpy() * c0.cpu().numpy()) + 1) / h
    bad = (np.abs(got - want) > tol) & vis
    assert bad.mean() < 1e-3, (bad.mean(), np.abs(got - want)[vis].max())
    assert active[vis].mean() > 0.5


# ---------------------------------------------------------------- 2. renders: the flag is the opacity only
def _eff_opacity(scene, c, opac=None, **kw):
    """The record's opacity o h of a flag-on forward with opacities ``opac`` (culled Gaussians keep o: never read)."""
    lib = _lib.load()
    o_in = torch.as_tensor(scene.opacity, device=DEV).reshape(-1, 1) if opac is None else opac.reshape(-1, 1)
    with torch.no_grad():
        _, (R, _, radii, geom, binning, img, *_) = _native_forward(scene, c, True, opac=o_in.contiguous(), **kw)
        torch.cuda.synchronize()
        s = read_state(lib, scene.P, R[0], c.image_width, c.image_height, geom[0], binning[0], img[0])
    o = s["conic_opacity"][:, 3:4].clone()
    vis = radii[0] > 0
    o[~vis] = o_in[~vis]
    return o.contiguous()


@pytest.mark.parametrize("case", ["rgb_depth", "rgb_exp_alpha", "c37", "c256", "joint", "lift"])
def test_render_is_the_flag_off_render_at_the_effective_opacity(case):
    scene = make_scene(60000, seed=4, sh=True, scale_mean=0.006)
    # the lift's sums are added per tile: a one-tile image gives each Gaussian one weight-sum partial
    c = orbit_cameras(4, 16, 16, fovx_deg=20.0)[2] if case == "lift" else orbit_cameras(4, 320, 224)[2]
    cam = _cam(c)
    pc, _ = _model(scene, grad=False)
    # the model's activated tensors, exactly as the renders pass them
    scene.xyz, scene.scales, scene.rotations = (pc.get_xyz.detach().cpu().numpy(), pc.get_scaling.detach().cpu().numpy(),
                                                pc.get_rotation.detach().cpu().numpy())
    o_eff = _eff_opacity(scene, c, opac=pc.get_opacity.detach())
    pc_eff = copy.copy(pc)   # the same parameter tensors, with the effective opacities
    pc_eff.__class__ = type("Eff", (GaussianModel,), {"get_opacity": property(lambda self: o_eff)})
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    with torch.no_grad():
        if case in ("rgb_depth", "rgb_exp_alpha"):
            fn = render if case == "rgb_depth" else render_with_depth
            a, b = fn(cam, pc, AAPipe(), bg), fn(cam, pc_eff, Pipe(), bg)
            keys = ["render", "depth", "radii"] + (["expected_depth", "alpha"] if case == "rgb_exp_alpha" else [])
        elif case in ("c37", "c256"):
            C = int(case[1:])
            f = torch.rand((scene.P, C), device=DEV, generator=_gen(5))
            kw = dict(num_channels=C, override_color=f)
            a, b = render_chn(cam, pc, AAPipe(), torch.zeros(C, device=DEV), **kw), \
                render_chn(cam, pc_eff, Pipe(), torch.zeros(C, device=DEV), **kw)
            keys = ["render", "radii"]
        elif case == "joint":
            f = torch.rand((scene.P, 64), device=DEV, generator=_gen(6))
            a = render_with_features(cam, pc, AAPipe(), bg, f, torch.zeros(64, device=DEV))
            b = render_with_features(cam, pc_eff, Pipe(), bg, f, torch.zeros(64, device=DEV))
            keys = ["render", "depth", "features", "radii"]
        else:
            maps = [torch.rand((16, 16, 16), device=DEV, generator=_gen(7)).half()]
            out = []
            for model, pipe in ((pc, AAPipe()), (pc_eff, Pipe())):
                fs, ws = torch.zeros((scene.P, 16), device=DEV), torch.zeros(scene.P, device=DEV)
                lift_views(model, [cam], maps, pipe, fs, ws)
                out.append(dict(feat=fs, weight=ws))
            a, b = out
            keys = ["weight"]
            assert a["weight"].abs().sum() > 0
            # the dL/dfeature contraction splits a tile's channels and pixels: its sums are equal up to their order
            assert torch.allclose(a["feat"], b["feat"], rtol=1e-5, atol=1e-6 * float(b["feat"].abs().max()))
    for k in keys:
        assert torch.equal(a[k], b[k]), k
    if case == "rgb_depth":   # and the flag matters on this scene
        assert not torch.equal(a["render"], render(cam, pc, Pipe(), bg)["render"])


# ---------------------------------------------------------------- 3. per-Gaussian gradients against float64
FAMILIES = {"subpixel": dict(scale_mean=0.004), "anisotropic": dict(scale_mean=0.02, aniso=True),
            "sideways": dict(scale_mean=0.02, sideways=True), "cov3D_precomp": dict(scale_mean=0.008, cov=True),
            "sh": dict(scale_mean=0.008, sh=True)}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_gradients_match_float64(family):
    f = FAMILIES[family]
    scene = make_scene(40000, seed=8, sh=True, scale_mean=f["scale_mean"])
    c = orbit_cameras(4, 256, 176)[0]
    if f.get("aniso"):
        rng = np.random.default_rng(9)
        scene.scales[:] *= (10 ** rng.uniform(-1.5, 1.5, scene.scales.shape)).astype(np.float32)
    if f.get("sideways"):
        push_sideways(scene, c, "xy", every=5)
    P = scene.P
    cov = None
    if f.get("cov"):
        cov = ar.cov6_from_factors(torch.as_tensor(scene.scales, device=DEV).double(),
                                   torch.as_tensor(scene.rotations, device=DEV).double()).float().contiguous()
    sh = bool(f.get("sh"))
    colors = None if sh else torch.rand((P, 3), device=DEV, generator=_gen(10))
    o_eff = _eff_opacity(scene, c, cov=cov, sh=sh, colors=colors)
    dout = torch.randn((3, c.image_height, c.image_width), device=DEV, generator=_gen(11))
    res = {}
    for aa, o in ((True, None), (False, o_eff)):
        native, (R, _, radii, geom, binning, img, *_) = _native_forward(scene, c, aa, opac=o, cov=cov, sh=sh,
                                                                       colors=colors)
        g = rasterizer._backward("t", native, radii, [dout], geom, R, binning, img)
        res[aa] = [x[0] if isinstance(x, list) else x for x in g]
        res[aa].append(radii[0] > 0)
    # order: means2D, colors, opacity, means3D, cov3D, sh, scales, rotations
    on, off = res[True], res[False]
    vis = on[-1]
    g_hat = off[2].reshape(-1).double()
    o = torch.as_tensor(scene.opacity, device=DEV).reshape(-1).double()
    h = (o_eff.reshape(-1).double() / o)
    want_op = h * g_hat
    assert torch.allclose(on[2].reshape(-1).double()[vis], want_op[vis], rtol=1e-5,
                          atol=1e-6 * float(want_op.abs().max()))
    # the float64 term: d(g_r r)/d(means3D, cov3D [, scales, rotations]) with g_r = o g / (2 h) where r > eps
    xyz = torch.as_tensor(scene.xyz, device=DEV).double().requires_grad_(True)
    if cov is None:
        sc = torch.as_tensor(scene.scales, device=DEV).double().requires_grad_(True)
        rq = torch.as_tensor(scene.rotations, device=DEV).double().requires_grad_(True)
        S6 = ar.cov6_from_factors(sc, rq)
        S6.retain_grad()
    else:
        S6 = cov.double().requires_grad_(True)
    tx, ty = math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5)
    a0, b, c0 = ar.screen_cov0(xyz, S6, np.asarray(c.world_view_transform).reshape(-1), c.image_width,
                               c.image_height, tx, ty)
    r = ar.r_torch(a0, b, c0)
    g_r = torch.where((r > ar.EPS) & vis, o * g_hat / (2 * h), torch.zeros_like(r)).detach()
    (g_r * r).sum().backward()
    pairs = [("means3D", on[3], off[3], xyz.grad), ("cov3D", on[4], off[4], S6.grad)]
    if cov is None:
        pairs += [("scales", on[6], off[6], sc.grad), ("rotations", on[7], off[7], rq.grad)]
    for name, a, b_, want in pairs:
        a, b_ = a.double(), b_.double()
        mag = torch.maximum(a.abs(), b_.abs()).amax(1, keepdim=True) + want.abs().amax(1, keepdim=True)
        bad = ((a - b_ - want).abs() > 2e-3 * mag).any(1) & vis
        assert bad.float().mean() < 0.01, (name, bad.float().mean())
        assert want[vis].abs().max() > 0, name


# ---------------------------------------------------------------- 4. camera gradients
def _leaf_grads(leaves):
    out = [torch.zeros_like(t) if t.grad is None else t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    return out


def test_camera_gradients_reproducible_and_change_nothing_else():
    """One-tile image (16 x 16), where every Gaussian has one blend partial: two identical backward passes agree
    bitwise, so what is compared is the geometry backward alone."""
    scene = make_scene(30000, seed=31, sh=True, scale_mean=0.01)
    pc, leaves = _model(scene)
    c = orbit_cameras(4, 16, 16, fovx_deg=20.0)[2]
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)

    def step(cam_grad):
        cam = _cam(c, cam_grad)
        o = render_with_depth(cam, pc, AAPipe(), bg)
        (o["render"].square().sum() + o["expected_depth"].square().sum()).backward()
        g = _leaf_grads(leaves)
        return g, (torch.cat([cam.world_view_transform.grad.reshape(-1), cam.full_proj_transform.grad.reshape(-1),
                              cam.camera_center.grad.reshape(-1)]) if cam_grad else None)

    g0, _ = step(False)
    g0b, _ = step(False)
    assert all(torch.equal(a, b) for a, b in zip(g0, g0b))
    g1, c1 = step(True)
    g2, c2 = step(True)
    assert all(torch.equal(a, b) for a, b in zip(g0, g1))
    assert torch.equal(c1, c2) and c1.abs().sum() > 0


def test_rigid_motion_identity():
    """dL/dtau of the pose correction at delta = 0 is W sum_i dL/dp_i (a camera translation is every Gaussian moved
    the other way), with the anti-aliasing term in both sides."""
    scene = make_scene(30000, seed=21, sh=True, scale_mean=0.006)
    c = orbit_cameras(4, 192, 128)[1]
    pc, _ = _model(scene, grad=False)
    pc._xyz.requires_grad_(True)
    pose = CameraPoseCorrection(1, DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    target = torch.rand((3, 128, 192), device=DEV, generator=_gen(4))
    img = render(pose(_cam(c), 0), pc, AAPipe(), bg)["render"]
    ((img - target) ** 2).sum().backward()
    g_tau = pose.delta.grad[0, 3:].double().cpu()
    Rw = torch.as_tensor(c.world_view_transform, dtype=torch.float64).T[:3, :3]
    gp = pc._xyz.grad.double().cpu()
    want = Rw @ gp.sum(0)
    assert ((g_tau - want).abs() <= 1e-4 * (Rw.abs() @ gp.abs().sum(0))).all(), (g_tau, want)


def test_finite_differences_along_pose_directions():
    """As test_camera_grad_gpu.py's check of the same name (large smooth Gaussians on a grid, a smooth linear
    functional, central differences with step 1e-3, tolerance 6 % of the sum of |gradient|), with the flag on; at
    sigma about 3.7 px the opacity factor h is about 0.99 and varies with the pose."""
    scene = make_scene(35, seed=61, sh=True, scale_mean=0.05)
    c = orbit_cameras(4, 128, 96)[0]
    gx, gy = np.meshgrid(np.linspace(-0.75, 0.75, 7), np.linspace(-0.45, 0.45, 5))
    t = np.stack([gx.ravel(), gy.ravel(), 3.0 + 0.1 * np.arange(35)], 1)
    t[:, :2] *= t[:, 2:3] / 3.0
    _, view = view_space(scene, c)
    set_view_space(scene, t, view, np.ones(35, bool))
    scene.scales[:] = 0.1
    scene.opacity[:] = 0.3
    pc, _ = _model(scene, grad=False)
    cam = _cam(c)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    ys, xs = torch.meshgrid(torch.linspace(0, 1, 96, device=DEV), torch.linspace(0, 1, 128, device=DEV), indexing="ij")
    weight = torch.stack([xs, ys, 1.0 - 0.5 * (xs + ys)])
    pose = CameraPoseCorrection(1, DEV)
    f = lambda: (render(pose(cam, 0), pc, AAPipe(), bg)["render"] * weight).sum()  # noqa: E731
    f().backward()
    g = pose.delta.grad[0].clone()
    dirs = torch.randn((6, 6), device=DEV, generator=_gen(8))
    dirs /= dirs.norm(dim=1, keepdim=True)
    step, errs = 1e-3, []
    with torch.no_grad():
        for d in dirs:
            pose.delta[0] = step * d
            fp = f().double()
            pose.delta[0] = -step * d
            fm = f().double()
            pose.delta[0] = 0
            errs.append(float(((fp - fm) / (2 * step) - (g * d).sum().double()).abs()))
    ref = max(float(g.abs().sum()), 1e-6)
    assert max(errs) <= 0.06 * ref, (errs, ref)


# ---------------------------------------------------------------- 5. batch
def test_batch_is_its_single_views():
    scene = make_scene(30000, seed=12, sh=True, scale_mean=0.008)
    cs = orbit_cameras(4, 16, 16, fovx_deg=20.0)[:3]
    pc, leaves = _model(scene)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    outs = render_batch([_cam(c) for c in cs], pc, AAPipe(), bg)
    sum(o["render"].square().sum() for o in outs).backward()
    gb = _leaf_grads(leaves)
    singles = [render(_cam(c), pc, AAPipe(), bg) for c in cs]
    for o, s in zip(outs, singles):
        assert torch.equal(o["render"], s["render"]) and torch.equal(o["depth"], s["depth"])
    gs = []
    for o, s in zip(outs, singles):
        s["render"].square().sum().backward()
        gs.append(_leaf_grads(leaves))
        # per view, on a one-tile image: the screen-space gradient is bitwise the single view's
        assert torch.equal(o["viewspace_points"].grad, s["viewspace_points"].grad)
    # the leaves sum the views before (batch) or after (singles) the activations' chain rule: fp32 reassociation
    for a, *b in zip(gb, *gs):
        want = sum(b)
        assert torch.allclose(a, want, rtol=1e-5, atol=1e-6 * float(want.abs().max() + 1e-30))


# ---------------------------------------------------------------- 6. footprint across resolutions
@pytest.mark.parametrize("chn", [False, True])
def test_footprint_is_kept_at_every_resolution(chn):
    """Isolated low-opacity sub-pixel Gaussians on a grid, rendered at 1x, 1/2x and 1/4x of 512 x 512 over background
    0 (alpha plane: 1 - final T; C > 4 path: a constant-1 feature).  With the flag the summed plane is o 2 pi
    sqrt(det C0) at every scale (within 3 %: what the 1/255 alpha floor and the 3 sigma cut-off drop); without it,
    o 2 pi sqrt(det C), which exceeds the undilated footprint by 2x or more at 1/4x."""
    n = 8
    scene = make_scene(n * n, seed=70, sh=True, scale_mean=0.01)
    c = orbit_cameras(4, 512, 512, fovx_deg=40.0)[0]
    gx, gy = np.meshgrid(np.linspace(-0.8, 0.8, n), np.linspace(-0.8, 0.8, n))
    t = np.stack([gx.ravel(), gy.ravel(), np.full(n * n, 4.0)], 1)
    t[:, :2] *= 4.0 * math.tan(c.FoVx * 0.5)
    _, view = view_space(scene, c)
    set_view_space(scene, t, view, np.ones(n * n, bool))
    scene.scales[:] = 0.012   # sigma about 2 px at 512, 0.5 px at 128
    scene.opacity[:] = 0.5
    pc, _ = _model(scene, grad=False)
    for k in (1, 2, 4):
        cam = _cam(c)
        cam.image_width = cam.image_height = 512 // k
        W = H = 512 // k
        tx = math.tan(c.FoVx * 0.5)
        a0, b, c0 = ar.screen_cov0(torch.as_tensor(scene.xyz, device=DEV).double(),
                                   ar.cov6_from_factors(torch.as_tensor(scene.scales, device=DEV).double(),
                                                        torch.as_tensor(scene.rotations, device=DEV).double()),
                                   np.asarray(c.world_view_transform).reshape(-1), W, H, tx, tx)
        a0, b, c0 = (x.cpu().numpy() for x in (a0, b, c0))
        want = ar.footprint(scene.opacity.reshape(-1), a0, b, c0).sum()
        dilated = ar.footprint(scene.opacity.reshape(-1), a0 + 0.3, b, c0 + 0.3).sum()
        got = {}
        with torch.no_grad():
            for pipe in (AAPipe(), Pipe()):
                if chn:
                    o = render_chn(cam, pc, pipe, torch.zeros(8, device=DEV), num_channels=8,
                                   override_color=torch.ones((scene.P, 8), device=DEV))
                    got[pipe.antialiasing] = float(o["render"][5].double().sum())
                else:
                    o = render_with_depth(cam, pc, pipe, torch.zeros(3, device=DEV))
                    got[pipe.antialiasing] = float(o["alpha"].double().sum())
        assert abs(got[True] / want - 1) < 0.03, (k, got[True], want)
        assert abs(got[False] / dilated - 1) < 0.03, (k, got[False], dilated)
        if k == 4:
            assert got[False] >= 2 * want, (got[False], want)
