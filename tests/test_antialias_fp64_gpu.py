"""Anti-aliased rasterization (sgb_view_inputs.antialiasing = 1: preprocess_kernel<true>, geom_backward_kernel<*, true>
and the blends reading the opacity o h) against the float64 restatements, per entry, through the C ABI:

  * geometry (tests/geom_ref.py with antialiasing): every case of test_geom_fp64_gpu.py with the flag on, where the
    record's opacity must be o h, its stored h the restatement's (sign = branch), dL_dopacity = h dL/d(o h) and the
    covariance term (o g / 2h) dr/dC0 must reach means3D, cov3D, scales and rotations within geom_ref.RTOL;
  * the families where anti-aliasing matters most, each asserting that it reached its branch:
      floor ......... det C0 / det C on both sides of the 2.5e-5 floor (sub-pixel Gaussians)
      needles ....... a0 c0 close to b^2: det C0 cancels (kappa0 > 1e3)
      b0 ............ an axis-aligned camera and axis-aligned Gaussians on the x = 0 plane: b = 0 exactly
      res_1/2/4 ..... one model rendered at 1x, 1/2x and 1/4x of one image size: more Gaussians near the floor
  * the blend with the flag on at C = 3, 5, 37, 256, 257, opaque and dense_faint_c65;
  * camera gradients (tests/camera_ref.py's fifth path) for every family of test_camera_grad_gpu.py, V = 1 and 3;
  * the lift (test_lift_gpu.py's check_lift) with the flag;
  * sensitivity: the floor case fails by at least 10x against each anti-aliasing mutation of the restatement and
    against a kernel that leaves dL_dopacity at g or makes it h^2 g.  The geometry comparison of dL_dopacity checks
    the kernel's stored h (g is recovered as dL_dopacity / |h|).  A wrong factor in dL_dopacity makes the recovered g
    wrong, so the covariance term (o g / 2h) dr/dC0 of every Gaussian above the floor disagrees with the kernel's;
    on the floor, where there is no such term, only the blend comparison (dL_dopacity against |h| times the blends'
    g) sees it.  The cases run with blend=False (anisotropic, needles, k2_size) have the first check only.

Tolerances are geom_ref.RTOL, camera_ref.RTOL and blend_ref.RTOL / ATOL_SCALE, unchanged; every case prints its
worst error ratio and fragile fractions (at most 2 %)."""
import math
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_ref  # noqa: E402
import geom_ref as gr  # noqa: E402
from raster_check import KERNEL_MUTATIONS, assert_ok, check_views, report  # noqa: E402
from scene_recipes import push_sideways, set_view_space, view_space  # noqa: E402
from test_camera_grad_gpu import FAMILIES, _native  # noqa: E402
from test_lift_gpu import check_lift  # noqa: E402

from semantic_gaussians_b200.scene_synth import (SynthCamera, look_at_camera, make_scene, orbit_cameras,  # noqa: E402
                                                 room_cameras)

pytestmark = pytest.mark.gpu

W0, H0 = 160, 96


def _bg(C):
    return np.linspace(0.05, 0.5, C).astype(np.float32)


def _run(name, scene, cams, **kw):
    t0 = time.time()
    res = check_views(scene, cams, _bg(3 if kw.get("sh_degree") is not None else scene.features.shape[1]),
                      antialiasing=True, **kw)
    report("aa", name, res, t0)
    assert_ok(res)
    return res


def _sh_scene(P=20000, seed=50, scale=0.02, kind="blob"):
    return make_scene(P, seed=seed, sh=True, scale_mean=scale, kind=kind)


def _cam(W=W0, H=H0, k=1):
    return orbit_cameras(4, W, H)[k]


# ---------------------------------------------------------------- the geometry cases of test_geom_fp64_gpu.py
@pytest.mark.parametrize("D,M", [(0, 16), (1, 16), (2, 16), (3, 16), (0, 1), (1, 4), (2, 9), (1, 9)])
def test_sh_degrees_and_coefficient_counts(D, M):
    _run(f"sh D={D} M={M}", _sh_scene(), [_cam()], sh_degree=D, M=M)


def test_sh_clamped_channels():
    scene = _sh_scene(seed=51)
    scene.shs[:, 0] *= 2.0
    res = _run("sh_clamped", scene, [_cam()], sh_degree=3)
    vis = res["radii"][0] > 0
    assert float(res["first_state"]["clamped"].cpu()[vis].double().mean()) >= 0.05


@pytest.mark.parametrize("axes", ["x", "y", "xy"])
def test_sideways_beyond_the_frustum_clamp(axes):
    scene = _sh_scene(seed=52, scale=0.03)
    cam = _cam()
    sel = push_sideways(scene, cam, axes)
    res = _run(f"sideways_{axes}", scene, [cam], sh_degree=3)
    t, _ = view_space(scene, cam)
    vis = res["radii"][0].numpy() > 0
    for ax in axes:
        k, tan = (0, math.tan(cam.FoVx * 0.5)) if ax == "x" else (1, math.tan(cam.FoVy * 0.5))
        assert (sel & vis & (np.abs(t[:, k] / t[:, 2]) > 1.3 * tan * 1.01)).sum() >= 20


def test_near_plane():
    scene = _sh_scene(seed=53, scale=0.01)
    cam = _cam()
    t, view = view_space(scene, cam)
    rng = np.random.default_rng(0)
    idx = np.arange(scene.P)
    near, culled = idx % 40 == 0, idx % 40 == 20
    scene.scales[near] *= 15.0
    for sel, lo, hi in ((near, 0.2001, 0.3), (culled, 0.1, 0.2)):
        z = rng.uniform(lo, hi, int(sel.sum()))
        t[sel, :2] *= (z / t[sel, 2])[:, None]
        t[sel, 2] = z
    set_view_space(scene, t, view, near | culled)
    res = _run("near_plane", scene, [cam], sh_degree=3)
    r = res["radii"][0].numpy()
    assert (r[near] > 0).sum() > 100 and r[near].max() > W0
    assert (r[culled] == 0).all()


def test_ragged_image_borders():
    _run("ragged_borders", _sh_scene(seed=54), [orbit_cameras(4, 173, 101, radius=2.0)[2]], sh_degree=3)


def test_anisotropic_and_subpixel_gaussians():
    scene = _sh_scene(seed=55, scale=0.03)
    i = np.arange(scene.P)
    # test_geom_fp64_gpu.py's needles are 3e-4 and its pancakes 1e-4 thin; with the filter, 95 % of those needles
    # have det C0 / det C within fp32 rounding of the 2.5e-5 floor (det C0 cancels to below its own rounding
    # error), so which branch they take is not decided by the arithmetic and they would all be left out as fragile.
    # 2e-3 keeps the ratio 150 and kappa0 above 1e4 with the decision resolved.
    scene.scales[i % 4 == 0] = np.array([0.3, 2e-3, 2e-3], np.float32)
    scene.scales[i % 4 == 1] = np.array([0.1, 0.1, 2e-3], np.float32)
    scene.scales[i % 4 == 2] = 5e-4
    # geometry only, as in test_geom_fp64_gpu.py (the blend restatement flags too many pixels as fragile here)
    _run("anisotropic", scene, [_cam()], sh_degree=3, blend=False)


def test_unnormalised_quaternions():
    scene = _sh_scene(seed=56)
    q = scene.rotations
    q[:, 0] = -np.abs(q[:, 0])
    q *= np.linspace(0.5, 2.0, scene.P, dtype=np.float32)[:, None]
    _run("quat_unnormalised", scene, [_cam()], sh_degree=3)


@pytest.mark.parametrize("mod", [0.6, 1.7])
def test_scale_modifier(mod):
    _run(f"mod{mod}", _sh_scene(seed=57), [_cam()], sh_degree=3, scale_modifier=mod)


def test_cov3d_precomp():
    scene = _sh_scene(seed=58)
    cam = _cam()
    q = scene.rotations * np.linspace(0.5, 2.0, scene.P, dtype=np.float32)[:, None]
    f = gr.geom_forward(scene.xyz, scene.opacity, cam.world_view_transform, cam.full_proj_transform,
                        cam.camera_center, W0, H0, cam.tanfovx, cam.tanfovy, scales=scene.scales, rotations=q)
    _run("cov3D_precomp", scene, [cam], sh_degree=3, cov3D_precomp=f["cov3D"].v.numpy().astype(np.float32))


@pytest.mark.parametrize("C", [3, 32])
def test_colors_precomp(C):
    _run(f"colors_c{C}", make_scene(20000, seed=59, channels=C), [_cam()])


def test_room_camera_inside_the_cloud():
    _run("room", _sh_scene(P=60000, seed=60, kind="room"), [room_cameras(3, W0, H0)[0]], sh_degree=3)


def test_sh_batch_with_own_dcolors():
    res = _run("batch_sh", _sh_scene(seed=61), orbit_cameras(3, W0, H0), sh_degree=3, seed=4)
    assert len(res["radii"]) == 3


@pytest.mark.parametrize("what,offset", [("rotations", 4), ("dL_drotations", 8), ("means3D", 12), ("scales", 4),
                                         ("shs", 8)])
def test_unaligned_per_gaussian_arrays(what, offset):
    _run(f"layout_{what}+{offset}", _sh_scene(seed=63), [_cam()], sh_degree=3, offsets={what: offset})


@pytest.mark.parametrize("P,W,H", [(10000, 256, 256), (20000, 320, 240)])
def test_calibration_configurations(P, W, H):
    t0 = time.time()
    res = check_views(make_scene(P, seed=2, sh=True), [orbit_cameras(4, W, H)[1]],
                      np.linspace(0.0, 0.5, 3).astype(np.float32), seed=5, sh_degree=3, antialiasing=True)
    report("aa", f"calibration P={P} {W}x{H} SH", res, t0)
    assert_ok(res)


def test_k2_size_scene():
    _run("k2_size", make_scene(1_000_000, seed=0, sh=True), [orbit_cameras(4, 1920, 1080)[1]], sh_degree=3,
         blend=False)


# ---------------------------------------------------------------- where anti-aliasing matters most
def _visible_ok(res):
    f = res["geom"]
    return f, f["visible"] & ~f["fragile"]


def _floor_scene():
    """Every other Gaussian sub-pixel (scales 10^-4.5 .. 10^-2.5): det C0 / det C on both sides of the floor."""
    scene = _sh_scene(seed=70)
    i = np.arange(scene.P)
    rng = np.random.default_rng(70)
    scene.scales[i % 2 == 0] = (10 ** rng.uniform(-4.5, -2.5, (int((i % 2 == 0).sum()), 3))).astype(np.float32)
    return scene


def test_floor_both_sides():
    f, ok = _visible_ok(_run("floor", _floor_scene(), [_cam()], sh_degree=3))
    above, below = int((ok & f["aa_active"]).sum()), int((ok & ~f["aa_active"]).sum())
    print(f"{above} Gaussians above the floor, {below} on it")
    assert above >= 1000 and below >= 1000


def test_needles_with_cancelling_det_c0():
    scene = _sh_scene(seed=71, scale=0.03)
    i = np.arange(scene.P)
    n = int((i % 8 == 0).sum())
    rng = np.random.default_rng(71)
    scene.scales[i % 8 == 0] = np.array([0.3, 2e-3, 2e-3], np.float32) * rng.uniform(0.5, 2, (n, 1)).astype(np.float32)
    # geometry only: the blend restatement flags about 4 % of the pixels of this scene as fragile
    f, ok = _visible_ok(_run("needles", scene, [_cam()], sh_degree=3, blend=False))
    a0, b, c0 = (f["aa_cov0"].v[:, j] for j in range(3))
    kappa0 = ((a0 * c0).abs() + b * b) / (a0 * c0 - b * b).abs()
    k = int((ok & f["aa_active"] & (kappa0 > 1e3)).sum())
    print(f"{k} needles above the floor with kappa0 > 1e3 (max {float(kappa0[ok & f['aa_active']].max()):.3g})")
    assert k >= 100


def _axis_aligned_camera(W, H):
    """Looking along +y from (0, -3, 0): its rotation is a signed permutation, built exactly (no inverse)."""
    c = look_at_camera((0.0, -3.0, 0.0), (0.0, 0.0, 0.0), W, H)
    wvt = np.zeros((4, 4), np.float64)
    wvt[0, 0], wvt[2, 1], wvt[1, 2], wvt[3, 2], wvt[3, 3] = 1.0, -1.0, 1.0, 3.0, 1.0   # t = (x, -z, y + 3)
    proj = np.asarray(c.projection_matrix, np.float64)
    return SynthCamera(W, H, c.FoVx, c.FoVy, wvt.astype(np.float32), proj.astype(np.float32),
                       np.ascontiguousarray((wvt @ proj).astype(np.float32)),
                       np.array([0.0, -3.0, 0.0], np.float32))


def test_axis_aligned_b_zero():
    scene = _sh_scene(seed=72)
    cam = _axis_aligned_camera(W0, H0)
    i = np.arange(scene.P)
    on = i % 2 == 0
    scene.xyz[on, 0] = 0.0                                    # t.x = 0: the Jacobian's first row has no z term
    scene.rotations[on] = np.array([1.0, 0.0, 0.0, 0.0], np.float32)   # diagonal world covariance
    f, ok = _visible_ok(_run("b0", scene, [cam], sh_degree=3))
    b = f["aa_cov0"].v[:, 1]
    n = int((ok & torch.as_tensor(on, device=b.device) & (b == 0) & f["aa_active"]).sum())
    print(f"{n} visible Gaussians with b = 0 exactly")
    assert n >= 1000


@pytest.mark.parametrize("div", [1, 2, 4])
def test_one_model_at_three_image_sizes(div):
    res = _run(f"res_1/{div}", _sh_scene(seed=73, scale=0.01), [_cam(320 // div, 192 // div)], sh_degree=3)
    f, ok = _visible_ok(res)
    print(f"1/{div}: {int((ok & ~f['aa_active']).sum())} of {int(ok.sum())} visible Gaussians on the floor")


# ---------------------------------------------------------------- the blend with the flag on
BLEND = {f"c{C}": (20000, C, 0.02, None) for C in (3, 5, 37, 256, 257)}
BLEND.update({"opaque": (4000, 32, 0.08, 0.999), "dense_faint_c65": (100000, 65, 0.05, 0.02)})


@pytest.mark.parametrize("name", list(BLEND))
def test_blend_matches_fp64(name):
    P, C, scale, opacity = BLEND[name]
    W, H = (128, 96) if name.startswith("dense") else (W0, H0)
    scene = make_scene(P, seed=40, channels=C, scale_mean=scale)
    if opacity is not None:
        scene.opacity[:] = opacity
    res = _run(f"blend_{name}", scene, [_cam(W, H)])
    if name == "dense_faint_c65":
        assert res["chunks"] > res["lens"].numel() * 8      # the pool's first guess overflowed and was retried


# ---------------------------------------------------------------- camera gradients
@pytest.mark.parametrize("V", [1, 3])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_camera_gradient_matches_float64(family, V):
    scene = make_scene(20000, seed=11, sh=True, scale_mean=0.02)
    cams = orbit_cameras(4, 160, 96)[:V]
    push_sideways(scene, cams[0], "xy", every=23)
    worst = 0.0
    for r in _native(scene, cams, antialiasing=True, **FAMILIES[family]):
        contrib, mag = camera_ref.camera_terms(*r["args"], **r["kw"], dev="cuda:0")
        worst = max(worst, camera_ref.check_sum(r["cam"], contrib, mag))
        if r["kw"]["shs"] is None:   # the opacity factor does not depend on the camera centre either
            assert not r["cam"][32:].any()
    print(f"\n[fp64 aa camera] {family} V={V}: {worst:.3g}")
    assert worst <= 1.0, worst


# ---------------------------------------------------------------- lift
def test_lift_matches_fp64():
    """sgb_lift_batch with the flag: the blend weights it lifts by use the opacity o h (test_lift_gpu.py's check_lift
    on the kernels' own state, an fp16 map of 65 channels past the first weight-pool item)."""
    scene = make_scene(20000, seed=50, channels=1, scale_mean=0.02)
    i = np.arange(scene.P)
    scene.scales[i % 4 == 0] *= 0.1                        # sub-pixel: h well below 1, some on the floor
    res = check_lift(scene, [_cam()], 65, torch.float16, antialiasing=True)
    print(f"\n[lift fp64 aa]: fragile={res['fragile']:.4%} " + " ".join(f"{k}={v:.3g}" for k, v in res["errs"].items()))
    assert res["fragile"] <= 0.02 and all(v <= 1.0 for v in res["errs"].values()), res
    st = res["states"][0]
    o = torch.as_tensor(scene.opacity, device=st["conic_opacity"].device).reshape(-1)
    seen = res["ws"] > 0
    assert float((st["conic_opacity"][seen, 3] < 0.99 * o[seen]).double().mean()) > 0.2   # the lift saw o h, not o


# ---------------------------------------------------------------- the comparison rejects anti-aliasing bugs
def test_comparison_rejects_anti_aliasing_bugs():
    """The floor case against each mutation of the restatement's anti-aliasing backward (geom_ref.AA_MUTATIONS) and
    against a kernel that writes g or h^2 g into dL_dopacity instead of h g (raster_check.KERNEL_MUTATIONS, applied
    to the kernel's output): every one must exceed the tolerance by at least 10x in its worst entry."""
    factors = {}
    for mut in gr.AA_MUTATIONS + KERNEL_MUTATIONS:
        res = check_views(_floor_scene(), [_cam()], _bg(3), sh_degree=3, antialiasing=True, mutation=mut)
        name, worst = max(res["errs"].items(), key=lambda kv: kv[1])
        factors[mut] = (worst, name)
    print("\n[fp64 aa mutations] worst entry / tolerance: " +
          " ".join(f"{m}={x:.3g} ({n})" for m, (x, n) in factors.items()))
    assert all(x >= 10 for x, _ in factors.values()), factors
