"""The geometry kernels (preprocess_kernel in csrc/preprocess.cu, geom_backward_kernel in csrc/geom_bwd.cu with
csrc/geom_grad.cuh) against the float64 restatement (tests/geom_ref.py), per Gaussian, through the C ABI.  The
restatement's backward runs on the kernel's own cov3D and clamped flags and on the kernel blend's dL_dmeans2D,
dL_dconic and dL_dcolors (which tests/test_blend_fp64_gpu.py pins), so the only error measured is the geometry
kernels' own.  Every float entry must satisfy |got - want| <= geom_ref.RTOL * magnitude; integers must be equal;
only fragile Gaussians (at most 2 %) are left out.

Which case reaches which branch:
  sh D = 0..3, M = 16 / (D+1)^2 / 9 ... the degree branches of sh_basis / colour_grad; coefficients >= (D+1)^2 of
                                        dL_dsh must stay exactly 0 (their magnitude is 0)
  sh_clamped ......................... >= 5 % of colour channels clamped: the clamp mask on the RGB gradient
  sideways_x / _y / _xy .............. |t/tz| beyond 1.3 tan(fov / 2): pass_u / pass_v and the clamped Jacobian
  near_plane ......................... view z in (0.2, 0.3] (huge radii, rects clipped to the grid) and <= 0.2
                                       (culled: gradients exactly 0)
  ragged_borders ..................... W, H not multiples of 16, a close camera: rects clipped at every border
  anisotropic ........................ scale ratios up to 10^3 (needles, pancakes) and sub-pixel Gaussians
  quat_unnormalised .................. quaternion norms 0.5 - 2 and negative w: used as given, both ways
  mod0.6 / mod1.7 .................... the gradient w.r.t. the already-modified scale
  cov3D_precomp ...................... dL_dcov3D as the output; no scale / rotation writes
  colors_c3 / colors_c32 ............. the geometry backward fed by each blend family without SH
  room ............................... camera inside the cloud: large 1 / |v| in the SH direction gradient
  batch_sh ........................... V = 3 SH views with their own dL_dcolors: per-view SH geometry gradients
  shared_dcolors_sh .................. V = 3 SH views sharing one dL_dcolors: SGB_E_INVALID, nothing launched
  layout_* ........................... rotations, dL_drotations, means3D, scales, shs at +4, +8, +12 bytes
  calibration ........................ the scenes, cameras and backgrounds of the SH configurations of
                                       test_parity_gpu.py::test_backward_vs_reference, whose kernels are pinned to
                                       the compiled reference (the feature ones run in test_blend_fp64_gpu.py,
                                       whose check_views checks the geometry too).  dL/dout is drawn here, not the
                                       one the reference was run with
  k2_size ............................ 1 M Gaussians, 1920 x 1080, SH D = 3, every Gaussian checked

geom_ref.RTOL = 16 * 2^-24 was calibrated on the calibration configurations (see geom_ref.py): measured on an H100
80GB HBM3 at a 700 W power limit, the largest error there is 0.075 of the tolerance, and 0.10 across this file and
test_blend_fp64_gpu.py."""
import ctypes as Ct
import math
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import geom_ref as gr  # noqa: E402
from raster_check import DEV, assert_ok, check_views, report  # noqa: E402
from scene_recipes import push_sideways, set_view_space, view_space  # noqa: E402
from util import dev_cam, dev_scene  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras, room_cameras  # noqa: E402

pytestmark = pytest.mark.gpu

W0, H0 = 160, 96


def _bg(C):
    return np.linspace(0.05, 0.5, C).astype(np.float32)


def _run(name, scene, cams, **kw):
    t0 = time.time()
    res = check_views(scene, cams, _bg(3 if kw.get("sh_degree") is not None else scene.features.shape[1]), **kw)
    report("geom", name, res, t0)
    assert_ok(res)
    return res


def _sh_scene(P=20000, seed=50, scale=0.02, kind="blob"):
    return make_scene(P, seed=seed, sh=True, scale_mean=scale, kind=kind)


@pytest.mark.parametrize("D,M", [(0, 16), (1, 16), (2, 16), (3, 16), (0, 1), (1, 4), (2, 9), (1, 9)])
def test_sh_degrees_and_coefficient_counts(D, M):
    _run(f"sh D={D} M={M}", _sh_scene(), [orbit_cameras(4, W0, H0)[1]], sh_degree=D, M=M)


def test_sh_clamped_channels():
    scene = _sh_scene(seed=51)
    scene.shs[:, 0] *= 2.0          # DC in (-3, 3): C0 dc + 0.5 < 0 for dc < -1.77
    res = _run("sh_clamped", scene, [orbit_cameras(4, W0, H0)[1]], sh_degree=3)
    vis = res["radii"][0] > 0
    frac = float(res["first_state"]["clamped"].cpu()[vis].double().mean())
    print(f"clamped channels: {frac:.2%}")
    assert frac >= 0.05


@pytest.mark.parametrize("axes", ["x", "y", "xy"])
def test_sideways_beyond_the_frustum_clamp(axes):
    scene = _sh_scene(seed=52, scale=0.03)
    cam = orbit_cameras(4, W0, H0)[1]
    sel = push_sideways(scene, cam, axes)
    res = _run(f"sideways_{axes}", scene, [cam], sh_degree=3)
    t, _ = view_space(scene, cam)
    vis = res["radii"][0].numpy() > 0
    for ax in axes:
        k, tan = (0, math.tan(cam.FoVx * 0.5)) if ax == "x" else (1, math.tan(cam.FoVy * 0.5))
        beyond = sel & vis & (np.abs(t[:, k] / t[:, 2]) > 1.3 * tan * 1.01)
        print(f"axis {ax}: {int(beyond.sum())} clamped Gaussians survive the cull")
        assert beyond.sum() >= 20


def test_near_plane():
    scene = _sh_scene(seed=53, scale=0.01)
    cam = orbit_cameras(4, W0, H0)[1]
    t, view = view_space(scene, cam)
    rng = np.random.default_rng(0)
    idx = np.arange(scene.P)
    near, culled = idx % 40 == 0, idx % 40 == 20
    scene.scales[near] *= 15.0                      # tens to hundreds of pixels at z = 0.2 .. 0.3
    for sel, lo, hi in ((near, 0.2001, 0.3), (culled, 0.1, 0.2)):
        z = rng.uniform(lo, hi, int(sel.sum()))
        t[sel, :2] *= (z / t[sel, 2])[:, None]     # same direction from the camera, nearer
        t[sel, 2] = z
    set_view_space(scene, t, view, near | culled)
    res = _run("near_plane", scene, [cam], sh_degree=3)
    r = res["radii"][0].numpy()
    assert (r[near] > 0).sum() > 100 and r[near].max() > W0   # huge radii, rects clipped to the grid
    assert (r[culled] == 0).all()


def test_ragged_image_borders():
    W, H = 173, 101
    scene = _sh_scene(seed=54)
    res = _run("ragged_borders", scene, [orbit_cameras(4, W, H, radius=2.0)[2]], sh_degree=3)
    f = res["geom"]
    vis = f["visible"] & ~f["fragile"]
    px, r = f["means2D"].v, f["radii"].double()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    clipped = dict(left=px[:, 0] - r < 0, top=px[:, 1] - r < 0, right=torch.trunc((px[:, 0] + r + 15) / 16) > gx,
                   bottom=torch.trunc((px[:, 1] + r + 15) / 16) > gy)
    n = {k: int((c & vis).sum()) for k, c in clipped.items()}
    print(f"rects clipped per border: {n}")
    assert min(n.values()) >= 100     # every border clips rects; the right and bottom tiles are partial


def test_anisotropic_and_subpixel_gaussians():
    scene = _sh_scene(seed=55, scale=0.03)
    i = np.arange(scene.P)
    scene.scales[i % 4 == 0] = np.array([0.3, 3e-4, 3e-4], np.float32)     # needles, ratio 10^3
    scene.scales[i % 4 == 1] = np.array([0.1, 0.1, 1e-4], np.float32)      # pancakes
    scene.scales[i % 4 == 2] = 5e-4                                        # sub-pixel: the 0.3 floor dominates
    # geometry only: on this scene the blend restatement flags about 5 % of the pixels as fragile, more than its
    # comparison may leave out, so the blend is not compared here
    res = _run("anisotropic", scene, [orbit_cameras(4, W0, H0)[1]], sh_degree=3, blend=False)
    f = res["geom"]
    vis = f["visible"] & ~f["fragile"]
    k = f["conic"].v      # the eigenvalue ratio of the 2-D covariance, from its inverse
    mid = 0.5 * (k[:, 0] + k[:, 2])
    s = (mid * mid - (k[:, 0] * k[:, 2] - k[:, 1] * k[:, 1])).clamp(min=0).sqrt()
    ratio = (mid + s) / (mid - s)
    floor = vis & torch.as_tensor(i % 4 == 2, device=vis.device) & (f["radii"] == 3)
    print(f"max 2-D eigenvalue ratio {float(ratio[vis].max()):.3g}, max kappa {float(f['kappa'][vis].max()):.3g}, "
          f"{int(floor.sum())} sub-pixel Gaussians at the floor radius")
    assert float(ratio[vis].max()) > 1e3 and float(f["kappa"][vis].max()) > 1e3   # ill-conditioned 2-D covariances
    # sub-pixel: the covariance is the 0.3 low-pass, whose radius is ceil(3 sqrt(0.3 + sqrt(0.1))) = 3
    assert int(floor.sum()) >= 1000


def test_unnormalised_quaternions():
    scene = _sh_scene(seed=56)
    q = scene.rotations
    q[:, 0] = -np.abs(q[:, 0])                                             # negative w
    q *= np.linspace(0.5, 2.0, scene.P, dtype=np.float32)[:, None]
    _run("quat_unnormalised", scene, [orbit_cameras(4, W0, H0)[1]], sh_degree=3)


@pytest.mark.parametrize("mod", [0.6, 1.7])
def test_scale_modifier(mod):
    _run(f"mod{mod}", _sh_scene(seed=57), [orbit_cameras(4, W0, H0)[1]], sh_degree=3, scale_modifier=mod)


def test_cov3d_precomp():
    scene = _sh_scene(seed=58)
    cam = orbit_cameras(4, W0, H0)[1]
    q = scene.rotations * np.linspace(0.5, 2.0, scene.P, dtype=np.float32)[:, None]
    f = gr.geom_forward(scene.xyz, scene.opacity, cam.world_view_transform, cam.full_proj_transform,
                        cam.camera_center, W0, H0, cam.tanfovx, cam.tanfovy, scales=scene.scales, rotations=q)
    _run("cov3D_precomp", scene, [cam], sh_degree=3, cov3D_precomp=f["cov3D"].v.numpy().astype(np.float32))


@pytest.mark.parametrize("C", [3, 32])
def test_colors_precomp(C):
    scene = make_scene(20000, seed=59, channels=C)
    _run(f"colors_c{C}", scene, [orbit_cameras(4, W0, H0)[1]])


def test_room_camera_inside_the_cloud():
    scene = _sh_scene(P=60000, seed=60, kind="room")
    _run("room", scene, [room_cameras(3, W0, H0)[0]], sh_degree=3)


def test_sh_batch_with_own_dcolors():
    res = _run("batch_sh", _sh_scene(seed=61), orbit_cameras(3, W0, H0), sh_degree=3, seed=4)
    assert len(res["radii"]) == 3


def test_sh_batch_sharing_dcolors_is_rejected():
    """With shs, view v's geometry kernel reads dL_dcolors after view v's blend added into it: one buffer shared by
    the views would hand view v the colour gradients of views 0..v.  The call is refused before anything runs."""
    lib = _lib.load()
    scene = _sh_scene(P=2000, seed=62)
    cams = orbit_cameras(3, W0, H0)
    V, P = 3, scene.P
    sc = dev_scene(scene, DEV)
    bg = torch.zeros(3, device=DEV)
    inp = _lib.ViewInputs(P=P, D=3, M=16, W=W0, H=H0, C=3, background=bg.data_ptr(), means3D=sc["means3D"].data_ptr(),
                          shs=sc["shs"].data_ptr(), colors_precomp=None, opacities=sc["opacities"].data_ptr(),
                          scales=sc["scales"].data_ptr(), scale_modifier=1.0, rotations=sc["rotations"].data_ptr(),
                          cov3D_precomp=None, viewmatrix=None, projmatrix=None, campos=None, tan_fovx=0.0,
                          tan_fovy=0.0, prefiltered=0, debug=0)
    cms = [dev_cam(c, DEV) for c in cams]
    cam_arr = (_lib.Camera * V)(*[_lib.Camera(c["viewmatrix"].data_ptr(), c["projmatrix"].data_ptr(),
                                              c["campos"].data_ptr(), c["tanfovx"], c["tanfovy"]) for c in cms])
    ptrs = lambda ts: (Ct.c_void_p * V)(*[t.data_ptr() for t in ts])
    u8 = dict(dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    ctx = Ct.c_void_p()
    _lib.check(lib.sgb_ctx_create(Ct.byref(ctx), DEV.index), "sgb_ctx_create")
    try:
        radii = [torch.empty((P,), dtype=torch.int32, device=DEV) for _ in cams]
        geom = [torch.empty((lib.sgb_geometry_bytes(P),), **u8) for _ in cams]
        img = [torch.empty((lib.sgb_image_bytes(W0, H0),), **u8) for _ in cams]
        Rs = (Ct.c_int64 * V)()
        _lib.check(lib.sgb_forward_geometry_batch(ctx, Ct.byref(inp), V, cam_arr, ptrs(geom), ptrs(radii), Rs, stream))
        binning = [torch.empty((lib.sgb_binning_bytes(R),), **u8) for R in Rs]
        color = [torch.empty((3, H0, W0), device=DEV) for _ in cams]
        _lib.check(lib.sgb_forward_render_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(geom), ptrs(binning),
                                                ptrs(img), ptrs(radii), ptrs(color), None, stream))
        assert min(Rs) > 0
        dL = [torch.randn((3, H0, W0), device=DEV) for _ in cams]
        z = lambda *s: torch.zeros(s, device=DEV)
        shared = z(P, 3)
        grads = [dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 4), dL_dopacity=z(P), dL_dcolors=shared, dL_dmeans3D=z(P, 3),
                      dL_dcov3D=z(P, 6), dL_dsh=z(P, 16, 3), dL_dscales=z(P, 3), dL_drotations=z(P, 4))
                 for _ in cams]
        gr_arr = (_lib.ViewGrads * V)(*[_lib.ViewGrads(**{k: t.data_ptr() for k, t in g.items()}) for g in grads])
        torch.cuda.synchronize(DEV)
        launches = lib.sgb_ctx_launch_count(ctx, 0), lib.sgb_ctx_launch_count(ctx, 1)
        rc = lib.sgb_backward_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(radii), ptrs(geom), ptrs(binning),
                                    ptrs(img), ptrs(dL), gr_arr, stream)
        msg = lib.sgb_last_error()
        torch.cuda.synchronize(DEV)
        assert rc == -1, rc
        assert b"dL_dcolors" in msg, msg
        assert (lib.sgb_ctx_launch_count(ctx, 0), lib.sgb_ctx_launch_count(ctx, 1)) == launches
        for g in grads:
            assert all(float(t.abs().max()) == 0.0 for t in g.values())
    finally:
        torch.cuda.synchronize(DEV)
        lib.sgb_ctx_destroy(ctx)


@pytest.mark.parametrize("what", ["rotations", "dL_drotations", "means3D", "scales", "shs"])
@pytest.mark.parametrize("offset", [4, 8, 12])
def test_unaligned_per_gaussian_arrays(what, offset):
    _run(f"layout_{what}+{offset}", _sh_scene(seed=63), [orbit_cameras(4, W0, H0)[1]], sh_degree=3,
         offsets={what: offset})


@pytest.mark.parametrize("P,W,H", [(10000, 256, 256), (20000, 320, 240)])
def test_calibration_configurations(P, W, H):
    """The scenes, cameras and backgrounds of test_backward_vs_reference's SH configurations (scene seed 2, orbit
    camera 1, the background ramp), on which the kernels are pinned to the compiled reference.  dL/dout is drawn
    here (torch, on the device, zero at blend-fragile pixels), so the upstream gradients differ from the ones the
    reference was run with; the restatement runs on the kernels' own upstream gradients either way.  A failure
    here would mean the restatement or the tolerance is wrong."""
    scene = make_scene(P, seed=2, sh=True)
    t0 = time.time()
    res = check_views(scene, [orbit_cameras(4, W, H)[1]], np.linspace(0.0, 0.5, 3).astype(np.float32), seed=5,
                      sh_degree=3)
    report("geom", f"calibration P={P} {W}x{H} SH", res, t0)
    assert_ok(res)


def test_k2_size_scene():
    """1 M Gaussians at 1920 x 1080 with SH degree 3 (the K2 workload's size), every Gaussian checked; the blend
    restatement is skipped here (its own calibration cases cover the blend), the geometry runs in float64 on the
    device."""
    scene = make_scene(1_000_000, seed=0, sh=True)
    _run("k2_size", scene, [orbit_cameras(4, 1920, 1080)[1]], sh_degree=3, blend=False)
