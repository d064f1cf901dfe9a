"""Camera gradients on the GPU (sgb_backward_batch_cam / sgb_backward_joint_batch_cam, the autograd plumbing of
rasterizer.py and camera_opt.CameraPoseCorrection):

  1. per view against the float64 autograd restatement of tests/camera_ref.py, fed with the kernel's own per-Gaussian
     upstream gradients (dL_dmeans2D, dL_dconic, dL_dcolors) and forward state (cov3D, clamped): render families
     (SH / colours, scale-rotation / cov3D_precomp), render_chn with C = 3, 32 and 300 and the joint render, V = 1
     and 3; batches of 11 views (split at 8) give each view what a single-view call gives;
  2. the rigid-motion identity, exact in mathematics: moving the camera by delta is moving every Gaussian by the
     same motion in the camera frame, so at delta = 0 the pose gradient is the summed per-Gaussian gradients carried
     into the camera frame (translation with SH, rotation with colours); this covers the expected-depth path too,
     whose dL/dz stays inside the library;
  3. bitwise: per-Gaussian gradients with and without camera gradients, two identical backwards, rendering and
     lift_scene through CameraPoseCorrection at delta = 0;
  4. central differences along six random pose directions;
  5. pose recovery from perturbed cameras with the Gaussians frozen (RGB, 32-channel features, joint render);
  6. an empty scene and a view that sees nothing give zero camera gradients."""
import ctypes as Ct
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_ref  # noqa: E402
from raster_check import read_state  # noqa: E402
from scene_recipes import push_sideways  # noqa: E402

from semantic_gaussians_b200 import _lib, rasterizer  # noqa: E402
from semantic_gaussians_b200.camera_opt import CameraPoseCorrection, rotation  # noqa: E402
from semantic_gaussians_b200.fusion import lift_scene  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.loss_utils import photometric_loss  # noqa: E402
from semantic_gaussians_b200.renderer import (render, render_batch, render_chn, render_chn_batch,  # noqa: E402
                                              render_with_depth, render_with_features)
from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras, room_cameras  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


class CovPipe(Pipe):
    compute_cov3d_python = True


class Cam:
    pass


def _cam(c, grad=False):
    v = Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
    v.uid = 0
    for name in ("world_view_transform", "full_proj_transform", "camera_center", "projection_matrix"):
        setattr(v, name, torch.as_tensor(getattr(c, name), device=DEV).clone().requires_grad_(grad))
    return v


def _cam_grads(v):
    return torch.cat([v.world_view_transform.grad.reshape(-1), v.full_proj_transform.grad.reshape(-1),
                      v.camera_center.grad.reshape(-1)])


def _model(scene, sh_degree=3, grad=True):
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, scene.shs, device=DEV)
    pc.active_sh_degree = sh_degree
    leaves = [pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest]
    for t in leaves:
        t.requires_grad_(grad)
    return pc, leaves


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---------------------------------------------------------------- 1. against float64, per view (C ABI driver)
def _native(scene, cams, *, C=3, sh_degree=None, cov=False, joint_c=0, seed=0, antialiasing=False):
    """Forward through rasterizer._forward and backward through sgb_backward_[joint_]batch_cam with per-view gradient
    buffers the test owns; returns per view the camera gradient (35) and the inputs of camera_ref.camera_terms (with
    antialiasing also the raw opacities, the blends' dL/d(o h), recovered as dL_dopacity / |h|, and the branch the
    kernel took, the sign of h)."""
    lib = _lib.load()
    P = scene.P
    t = lambda a: torch.as_tensor(a, device=DEV).contiguous()  # noqa: E731
    xyz, opac = t(scene.xyz), t(scene.opacity)
    sh = t(scene.shs) if sh_degree is not None else None
    colors = None if sh is not None else torch.rand((P, C), device=DEV, generator=_gen(seed))
    scales = rots = cov3D = None
    if cov:
        pc, _ = _model(scene, grad=False)
        cov3D = pc.get_covariance(1.0).detach().contiguous()
    else:
        scales, rots = t(scene.scales), t(scene.rotations)
    feats = torch.randn((P, joint_c), device=DEV, generator=_gen(seed + 1)) if joint_c else None
    bgf = torch.linspace(0.0, 0.3, joint_c, device=DEV) if joint_c else None
    bg = torch.linspace(0.05, 0.5, C, device=DEV)
    W, H = cams[0].image_width, cams[0].image_height
    cl = [(t(c.world_view_transform), t(c.full_proj_transform), t(c.camera_center), math.tan(c.FoVx * 0.5),
           math.tan(c.FoVy * 0.5)) for c in cams]
    native, (R, color, radii, geom, binning, img, depth, _, _, *feat) = rasterizer._forward(
        bool(joint_c), "test", cl, bg, xyz, colors, opac, scales, rots, 1.0, cov3D, H, W, sh,
        sh_degree or 0, False, False, C, features=feats, bg_features=bgf, antialiasing=antialiasing)
    inp, cameras, _, _ = native
    V = len(cams)
    z = lambda *s: torch.zeros(s, device=DEV)  # noqa: E731
    M = sh.shape[1] if sh is not None else 0
    grads = [dict(m2=z(P, 3), conic=z(P, 4), opac=z(P), col=z(P, C), m3=z(P, 3), cov=z(P, 6), sh=z(P, max(M, 1), 3),
                  s=z(P, 3), r=z(P, 4)) for _ in range(V)]
    vg = (_lib.ViewGrads * V)(*[_lib.ViewGrads(*[g[k].data_ptr() for k in ("m2", "conic", "opac", "col", "m3", "cov")],
                                                g["sh"].data_ptr() if M else None, g["s"].data_ptr(),
                                                g["r"].data_ptr()) for g in grads])
    cam_out = z(V, 35)
    cg = (_lib.CameraGrads * V)(*[_lib.CameraGrads(cam_out[v].data_ptr(), cam_out[v, 16:].data_ptr(),
                                                   cam_out[v, 32:].data_ptr()) for v in range(V)])
    dout = [torch.randn(c_.shape, device=DEV, generator=_gen(seed + 10 + v)) for v, c_ in enumerate(color)]
    arr = lambda ts: (Ct.c_void_p * V)(*[x.data_ptr() for x in ts])  # noqa: E731
    stream, ctx = rasterizer._stream_ctx(DEV)
    common = (ctx, Ct.byref(inp), V, cameras, (Ct.c_int64 * V)(*R), arr(radii), arr(geom), arr(binning), arr(img),
              arr(dout), None, None, vg)
    if joint_c:
        gf = z(P, joint_c)
        dfeat = [torch.randn(f.shape, device=DEV, generator=_gen(seed + 30 + v)) for v, f in enumerate(feat[0])]
        rc = lib.sgb_backward_joint_batch_cam(*common, feats.data_ptr(), joint_c, bgf.data_ptr(), arr(dfeat),
                                              gf.data_ptr(), cg, stream)
    else:
        rc = lib.sgb_backward_batch_cam(*common, cg, stream)
    _lib.check(rc, "sgb_backward_batch_cam")
    torch.cuda.synchronize()
    out = []
    for v in range(V):
        st = read_state(lib, P, R[v], W, H, geom[v], binning[v], img[v], ("cov3D", "clamped", "aa_h"))
        c = cams[v]
        kw = dict(shs=sh, D=sh_degree or 0, clamped=st["clamped"], dL_dcolors=grads[v]["col"])
        if antialiasing:
            live = radii[v] > 0
            g_oh = torch.where(live, grads[v]["opac"].double() / st["aa_h"].abs().double().clamp(min=1e-30),
                               torch.zeros_like(grads[v]["opac"].double()))
            kw.update(antialiasing=True, opacities=opac.reshape(-1), dL_dopacity=g_oh, aa_active=st["aa_h"] > 0)
        out.append(dict(cam=cam_out[v].cpu(), args=(xyz, radii[v], cov3D if cov else st["cov3D"],
                                                    np.asarray(c.world_view_transform), np.asarray(c.full_proj_transform),
                                                    np.asarray(c.camera_center), W, H, math.tan(c.FoVx * 0.5),
                                                    math.tan(c.FoVy * 0.5), grads[v]["m2"], grads[v]["conic"]),
                        kw=kw, grads=grads[v]))
    return out


FAMILIES = {
    "sh_d3": dict(sh_degree=3), "sh_d1_cov": dict(sh_degree=1, cov=True), "colors_c3": dict(C=3),
    "colors_c3_cov": dict(C=3, cov=True), "chn_c32": dict(C=32), "chn_c300": dict(C=300),
    "joint_sh_c8": dict(sh_degree=3, joint_c=8), "joint_colors_c64": dict(C=3, joint_c=64),
}


@pytest.mark.parametrize("V", [1, 3])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_camera_gradient_matches_float64(family, V):
    scene = make_scene(20000, seed=11, sh=True, scale_mean=0.02)
    cams = orbit_cameras(4, 160, 96)[:V]
    push_sideways(scene, cams[0], "xy", every=23)     # frustum-clamped Gaussians in view 0
    worst = 0.0
    for v, r in enumerate(_native(scene, cams, **FAMILIES[family])):
        contrib, mag = camera_ref.camera_terms(*r["args"], **r["kw"], dev=DEV)
        worst = max(worst, camera_ref.check_sum(r["cam"], contrib, mag))
        if r["kw"]["shs"] is None:
            assert not r["cam"][32:].any()
    # camera_ref.RTOL = 16 * 2^-24 (see there)
    assert worst <= 1.0, worst


def test_batch_of_11_matches_single_views():
    """A batch past the native limit is split (8 + 3); every view's camera gradient is bitwise what a single-view
    render gives (on a one-tile image, where the upstream per-Gaussian gradients are reproducible)."""
    scene = make_scene(20000, seed=12, sh=True, scale_mean=0.02)
    pc, _ = _model(scene, grad=False)
    cams = [_cam(c, True) for c in orbit_cameras(11, 16, 16, fovx_deg=20.0)]   # one tile: see below
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    outs = render_batch(cams, pc, Pipe(), bg)
    sum(((o["render"] - 0.3) ** 2).sum() for o in outs).backward()
    batch = [_cam_grads(c) for c in cams]
    for c, want in zip(cams, batch):
        c2 = Cam()
        c2.__dict__.update({k: (x.detach().clone().requires_grad_(True) if isinstance(x, torch.Tensor) else x)
                            for k, x in c.__dict__.items()})
        ((render(c2, pc, Pipe(), bg)["render"] - 0.3) ** 2).sum().backward()
        assert torch.equal(_cam_grads(c2), want)
        assert want.abs().sum() > 0


# ---------------------------------------------------------------- 2. rigid-motion identity
@pytest.mark.parametrize("what", ["translation_sh", "rotation_colors", "translation_depth"])
def test_rigid_motion_identity(what):
    """p_cam' = R p_cam + tau is every Gaussian moved by W^T (p_cam' - p_cam) in the world with the camera fixed, so at
    delta = 0: dL/dtau = W sum_i dL/dp_i and dL/domega = sum_i [p_cam,i x (W dL/dp_i) + (the rotation term of
    dL/dcov3D_i)], p_cam,i = W p_i + t0.  With colours from SH the world-space view direction would not rotate with the
    Gaussians, so the rotation case uses colours without SH.  Both sides come from the same backward; the sums run in
    float64 and the tolerance is 1e-4 of the sum of |terms|."""
    scene = make_scene(30000, seed=21, sh=True, scale_mean=0.03)
    c = orbit_cameras(4, 192, 128)[1]
    cam = _cam(c)
    pose = CameraPoseCorrection(1, DEV)
    P = scene.P
    pc, _ = _model(scene, grad=False)
    xyz = torch.as_tensor(scene.xyz, device=DEV).requires_grad_(True)
    cov = pc.get_covariance(1.0).detach().requires_grad_(True)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    wrapped = pose(cam, 0)
    from semantic_gaussians_b200 import rgbd_rasterization as rr
    rs = rr.GaussianRasterizationSettings(image_height=128, image_width=192, tanfovx=math.tan(c.FoVx / 2),
                                          tanfovy=math.tan(c.FoVy / 2), bg=bg, scale_modifier=1.0,
                                          viewmatrix=wrapped.world_view_transform,
                                          projmatrix=wrapped.full_proj_transform, sh_degree=3,
                                          campos=wrapped.camera_center, prefiltered=False, debug=False)
    kw = dict(means3D=xyz, means2D=torch.zeros_like(xyz), opacities=pc.get_opacity.detach(), cov3D_precomp=cov)
    if what == "rotation_colors":
        kw["colors_precomp"] = torch.rand((P, 3), device=DEV, generator=_gen(3))
    else:
        kw["shs"] = pc.get_features.detach()
    rast = rr.GaussianRasterizer(rs)
    target = torch.rand((3, 128, 192), device=DEV, generator=_gen(4))
    if what == "translation_depth":
        img, radii, depth, E, A = rast.forward_expected_depth(**kw)
        loss = ((E - 2.0) ** 2).sum() + (A * target[:1]).sum()
    else:
        img, radii, depth = rast(**kw)
        loss = ((img - target) ** 2).sum()
    loss.backward()
    g_delta = pose.delta.grad[0].double().cpu()
    Wv = torch.as_tensor(c.world_view_transform, dtype=torch.float64).T[:3]          # W2C rows: [R | t0]
    Rw, t0 = Wv[:, :3], Wv[:, 3]
    gp = xyz.grad.double().cpu()
    want_tau = Rw @ gp.sum(0)
    tol_tau = 1e-4 * (Rw.abs() @ gp.abs().sum(0))
    assert ((g_delta[3:] - want_tau).abs() <= tol_tau).all(), (g_delta[3:], want_tau, tol_tau)
    if what == "rotation_colors":
        pcam = torch.as_tensor(scene.xyz, dtype=torch.float64) @ Rw.T + t0
        gcam = gp @ Rw.T
        # covariance: S_cam = R S R^T rotates by omega; dL/domega from dL/dS_cam = R dL/dS R^T
        g6 = cov.grad.double().cpu()
        G = torch.stack([torch.stack([g6[:, 0], g6[:, 1] / 2, g6[:, 2] / 2], 1),
                         torch.stack([g6[:, 1] / 2, g6[:, 3], g6[:, 4] / 2], 1),
                         torch.stack([g6[:, 2] / 2, g6[:, 4] / 2, g6[:, 5]], 1)], 1)
        c6 = cov.detach().double().cpu()
        S = torch.stack([torch.stack([c6[:, 0], c6[:, 1], c6[:, 2]], 1), torch.stack([c6[:, 1], c6[:, 3], c6[:, 4]], 1),
                         torch.stack([c6[:, 2], c6[:, 4], c6[:, 5]], 1)], 1)
        Gc, Sc = Rw @ G @ Rw.T, Rw @ S @ Rw.T
        Mx = 2.0 * Gc @ Sc                                   # dL/dK for S' = (I + K) S (I + K)^T at K = 0
        vee = torch.stack([Mx[:, 2, 1] - Mx[:, 1, 2], Mx[:, 0, 2] - Mx[:, 2, 0], Mx[:, 1, 0] - Mx[:, 0, 1]], 1)
        terms = torch.cat([torch.linalg.cross(pcam, gcam), vee], 0)
        want_w = terms.sum(0)
        tol_w = 1e-4 * terms.abs().sum(0)
        assert ((g_delta[:3] - want_w).abs() <= tol_w).all(), (g_delta[:3], want_w, tol_w)


# ---------------------------------------------------------------- 3. bitwise equalities
def _leaf_grads(leaves):
    out = [torch.zeros_like(t) if t.grad is None else t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    return out


# The blend backwards add each (Gaussian, tile) partial into the per-Gaussian gradients with a global reduction, so
# their order across tiles, and with it the last bits of dL_dmeans2D / dL_dconic / dL_dcolors, can change from run to
# run.  The bitwise comparisons below use a one-tile image (16 x 16), where every Gaussian has one partial, and at
# most 4 channels (the C > 4 contractions also split a tile): there two identical backward passes are first checked
# to agree bitwise, so what is compared is the geometry backward alone.
@pytest.mark.parametrize("fn", ["render", "render_with_depth", "render_chn", "render_with_features"])
def test_per_gaussian_gradients_unchanged_and_camera_gradients_reproducible(fn):
    scene = make_scene(30000, seed=31, sh=True, scale_mean=0.03)
    pc, leaves = _model(scene)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    feats = torch.randn((scene.P, 4), device=DEV, generator=_gen(2)).requires_grad_(True)
    c = orbit_cameras(4, 16, 16, fovx_deg=20.0)[2]

    def step(cam_grad):
        cam = _cam(c, cam_grad)
        if fn == "render":
            out = render(cam, pc, Pipe(), bg)["render"].square().sum()
        elif fn == "render_with_depth":
            o = render_with_depth(cam, pc, Pipe(), bg)
            out = o["expected_depth"].square().sum() + o["render"].sum()
        elif fn == "render_chn":
            o = render_chn(cam, pc, Pipe(), torch.zeros(4, device=DEV), num_channels=4, override_color=feats)
            out = o["render"].square().sum()
        else:
            o = render_with_features(cam, pc, Pipe(), bg, feats, torch.zeros(4, device=DEV))
            out = o["render"].square().sum() + o["features"].square().sum()
        out.backward()
        g = _leaf_grads(leaves + [feats]) if fn != "render" else _leaf_grads(leaves)
        return g, (_cam_grads(cam) if cam_grad else None)

    g0, _ = step(False)
    g0b, _ = step(False)
    assert all(torch.equal(a, b) for a, b in zip(g0, g0b)), "the one-tile backward is not reproducible"
    g1, c1 = step(True)
    g2, c2 = step(True)
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)
    assert torch.equal(c1, c2) and c1.abs().sum() > 0


def test_pose_module_at_zero_is_bitwise_the_camera():
    scene = make_scene(30000, seed=41, sh=True, scale_mean=0.03)
    pc, _ = _model(scene, grad=False)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    cams = [_cam(c) for c in orbit_cameras(3, 160, 112)]
    pose = CameraPoseCorrection(3, DEV)
    for i, cam in enumerate(cams):
        w = pose(cam, i)
        for name in ("world_view_transform", "full_proj_transform", "camera_center"):
            assert torch.equal(getattr(w, name).view(torch.int32), getattr(cam, name).view(torch.int32))
        a = render(cam, pc, Pipe(), bg)
        b = render(w, pc, Pipe(), bg)
        assert torch.equal(a["render"], b["render"]) and torch.equal(a["depth"], b["depth"])
    # lift_scene adds per-tile partials with a global reduction: on a one-tile map the sums are reproducible
    cams = [_cam(c) for c in orbit_cameras(3, 16, 16, fovx_deg=20.0)]
    C = 8
    maps = [torch.rand((C, 16, 16), device=DEV, generator=_gen(50 + i)) for i in range(3)]

    def lifted(views):
        with torch.no_grad():
            pc.create_semantic(C)
            r = lift_scene(pc, views, maps, Pipe(), every=1)
            return r["features"].clone(), r["weights"].clone()
    f1, w1 = lifted(cams)
    f1b, w1b = lifted(cams)
    assert torch.equal(f1, f1b) and torch.equal(w1, w1b), "lift_scene on one tile is not reproducible"
    f2, w2 = lifted([pose(cam, i) for i, cam in enumerate(cams)])
    assert torch.equal(f1, f2) and torch.equal(w1, w2) and bool((w1 > 0).any())


# ---------------------------------------------------------------- 4. finite differences
def test_finite_differences_along_pose_directions():
    """A fixed linear functional of the image of large, smooth Gaussians (weights that ramp smoothly across the
    image); central differences with step 1e-3 in float32 against the analytic directional derivative.  The Gaussians
    (sigma about 5.5 px) sit on a 7 x 5 grid facing the camera, 0.1 apart in depth, so that no pose step reorders them
    (a depth swap makes the image jump).  Opacity 0.3 puts the 1/255 alpha floor inside the 3-sigma footprint, so a
    footprint that gains or loses a tile adds or drops only zeros.  What the analytic gradient does not see is the
    pixels crossing the alpha floor: the reference's backward differentiates the smooth part only.  On this scene that
    part alone (the CPU restatement of the reference, world translations) differs from central differences by up to
    3 % of the sum of |gradient|; the tolerance is 6 %."""
    scene = make_scene(35, seed=61, sh=True, scale_mean=0.05)
    c = orbit_cameras(4, 128, 96)[0]
    gx, gy = np.meshgrid(np.linspace(-0.75, 0.75, 7), np.linspace(-0.45, 0.45, 5))
    t = np.stack([gx.ravel(), gy.ravel(), 3.0 + 0.1 * np.arange(35)], 1)
    t[:, :2] *= t[:, 2:3] / 3.0
    from scene_recipes import set_view_space, view_space
    _, view = view_space(scene, c)
    set_view_space(scene, t, view, np.ones(35, bool))
    scene.scales[:] = 0.15
    scene.opacity[:] = 0.3
    pc, _ = _model(scene, grad=False)
    cam = _cam(c)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    # smooth ramps: a random per-pixel weight would cancel the smooth part of the derivative over each footprint
    ys, xs = torch.meshgrid(torch.linspace(0, 1, 96, device=DEV), torch.linspace(0, 1, 128, device=DEV), indexing="ij")
    weight = torch.stack([xs, ys, 1.0 - 0.5 * (xs + ys)])
    pose = CameraPoseCorrection(1, DEV)
    f = lambda: (render(pose(cam, 0), pc, Pipe(), bg)["render"] * weight).sum()  # noqa: E731
    f().backward()
    g = pose.delta.grad[0].clone()
    dirs = torch.randn((6, 6), device=DEV, generator=_gen(8))
    dirs /= dirs.norm(dim=1, keepdim=True)
    h = 1e-3
    errs, scale = [], []
    with torch.no_grad():
        for d in dirs:
            pose.delta[0] = h * d
            fp = f().double()
            pose.delta[0] = -h * d
            fm = f().double()
            pose.delta[0] = 0
            fd = (fp - fm) / (2 * h)
            an = (g * d).sum().double()
            errs.append(float((fd - an).abs()))
            scale.append(float(an.abs()))
    ref = max(float(g.abs().sum()), 1e-6)
    assert max(errs) <= 0.06 * ref, (errs, scale, ref)


# ---------------------------------------------------------------- 5. pose recovery
# Set on an H100: 300 Adam steps from lr 2e-3 decaying to 1e-4 bring the seven or eight cameras that converge to
# 0.01 - 0.02 degrees and 0.01 - 0.03 mm.  The perturbation seed matters: with seeds 72 and 73 one camera of the eight
# (RGB loss) stops in a local minimum of the photometric loss at about 0.3 degrees and 8 mm.
POSE_STEPS, POSE_LR, POSE_LR_END, POSE_SCALE, POSE_SEED = 300, 2e-3, 1e-4, 0.03, 74


def _pose_error(est, true):
    """(rotation angle in degrees, translation in scene units) of est W2C relative to true."""
    Ee = est.world_view_transform.detach().double().T
    Et = true.world_view_transform.detach().double().T
    D = Ee @ torch.linalg.inv(Et)
    cosang = ((D[:3, :3].trace() - 1) / 2).clamp(-1, 1)
    return math.degrees(float(torch.arccos(cosang))), float(D[:3, 3].norm())


def _perturbed(cams, seed):
    rng = np.random.default_rng(seed)
    out = []
    for c in cams:
        axis = rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        d = rng.standard_normal(3)
        d /= np.linalg.norm(d)
        delta = torch.as_tensor(np.concatenate([axis * math.radians(1.0), d * 0.03]), dtype=torch.float32, device=DEV)
        moved = CameraPoseCorrection(1, DEV)
        with torch.no_grad():
            moved.delta[0] = delta
            w = moved(c, 0)
            p = Cam()
            p.__dict__.update(c.__dict__)
            p.world_view_transform = w.world_view_transform.detach().clone()
            p.full_proj_transform = w.full_proj_transform.detach().clone()
            p.camera_center = w.camera_center.detach().clone()
        out.append(p)
    return out


@pytest.mark.parametrize("target", ["rgb", "chn32", "joint"])
def test_pose_recovery(target):
    scene = make_scene(200_000, seed=71, kind="room", sh=True, scale_mean=POSE_SCALE)
    pc, _ = _model(scene, grad=False)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    feats = torch.randn((scene.P, 32), device=DEV, generator=_gen(9))
    true = [_cam(c) for c in room_cameras(8, 320, 240)]
    start = _perturbed(true, POSE_SEED)

    def images(cams):
        if target == "rgb":
            return [o["render"] for o in render_batch(cams, pc, Pipe(), bg)]
        if target == "chn32":
            return [o["render"] for o in render_chn_batch(cams, pc, Pipe(), torch.zeros(32, device=DEV), num_channels=32,
                                                          override_color=feats)]
        return [torch.cat([o["render"], o["features"]]) for o in
                [render_with_features(c, pc, Pipe(), bg, feats, torch.zeros(32, device=DEV)) for c in cams]]

    with torch.no_grad():
        gts = images(true)
    pose = CameraPoseCorrection(8, DEV)
    opt = torch.optim.Adam(pose.parameters(), lr=POSE_LR)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, (POSE_LR_END / POSE_LR) ** (1.0 / POSE_STEPS))
    e0 = [_pose_error(s, t) for s, t in zip(start, true)]
    for _ in range(POSE_STEPS):
        opt.zero_grad(set_to_none=True)
        imgs = images([pose(s, i) for i, s in enumerate(start)])
        sum(photometric_loss(im, gt)[0] for im, gt in zip(imgs, gts)).backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        e1 = [_pose_error(pose(s, i), t) for i, (s, t) in enumerate(zip(start, true))]
    for (r0, t0), (r1, t1) in zip(e0, e1):
        assert r1 <= r0 / 10 and t1 <= t0 / 10, (e0, e1)


# ---------------------------------------------------------------- 6. nothing to see
def test_empty_scene_and_empty_view_give_zero_camera_gradients():
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    scene = make_scene(2000, seed=81, sh=True, scale_mean=0.03)
    pc, leaves = _model(scene)
    away = look_at_camera((0.0, 0.0, 30.0), (0.0, 0.0, 60.0), 64, 48)      # looks away from the cloud
    cam = _cam(away, True)
    o = render(cam, pc, Pipe(), bg)
    assert not (o["radii"] > 0).any()
    (o["render"].sum() + leaves[0].sum() * 0).backward()
    assert not _cam_grads(cam).any()
    empty = make_scene(0, seed=82, sh=True)
    pc0, _ = _model(empty)
    cam = _cam(orbit_cameras(1, 64, 48)[0], True)
    for fn in (lambda c: render(c, pc0, Pipe(), bg)["render"],
               lambda c: render_with_features(c, pc0, Pipe(), bg, torch.zeros((0, 8), device=DEV, requires_grad=True),
                                              torch.zeros(8, device=DEV))["features"]):
        for t in (cam.world_view_transform, cam.full_proj_transform, cam.camera_center):
            t.grad = None
        (fn(cam).sum() + cam.world_view_transform.sum() * 0).backward()
        assert not _cam_grads(cam).any()
