"""Camera gradients without a GPU:

  * the per-Gaussian camera terms of semantic-gaussians_b200/csrc/geom_grad.cuh (project_grad's ProjectTerms,
    colour_grad's campos_grad, camera_grad), compiled for the host by g++ (tests/host/camera_grad_host.cpp), summed
    over a view and compared with the float64 autograd restatement of tests/camera_ref.py on seeded scenes with
    frustum-clamped and near-plane Gaussians, SH degrees 0-3, clamped colours and a dL/dz;
  * sgb_backward_batch_cam / sgb_backward_joint_batch_cam reject bad camera-gradient outputs before any CUDA call;
  * the pose correction module (camera_opt.py): R(omega), bitwise identity at delta = 0, its gradient, the camera
    centre and attribute delegation."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_ref  # noqa: E402
from scene_recipes import push_sideways, set_view_space, view_space  # noqa: E402

from oracle import oracle as orc  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.camera_opt import CameraPoseCorrection, rotation  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("camgrad") / "libcamgrad_host.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++",
                           "-I", os.path.join(ROOT, "semantic-gaussians_b200", "csrc"),
                           os.path.join(HERE, "host", "camera_grad_host.cpp"), "-o", out])
    lib = C.CDLL(out)
    lib.host_camera_grad.restype = None
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _scene(seed, deg, clamp, near):
    W, H = 160, 112
    scene = make_scene(4000, seed=seed, sh=True, scale_mean=0.08)
    cam = orbit_cameras(4, W, H)[seed % 4]
    if clamp:
        push_sideways(scene, cam, clamp)
    if near:   # every 7th Gaussian just beyond the near plane (z = 0.2), every 13th in front of it (culled)
        t, view = view_space(scene, cam)
        sel = np.arange(scene.P) % 7 == 3
        t[sel, 2] = np.linspace(0.21, 0.35, int(sel.sum()))
        t[sel, :2] *= 0.05
        cull = np.arange(scene.P) % 13 == 5
        t[cull, 2] = 0.1
        set_view_space(scene, t, view, sel | cull)
    f = orc.forward(orc.scene_dict(scene), orc.cam_dict(cam), W, H, np.zeros(3, np.float32), sh_degree=deg)
    return scene, cam, f["pre"], W, H


def _drop_fragile(pre, scene, cam):
    """radii with the Gaussians whose clamp decision lies within rounding of its threshold set to 0 (both sides
    then leave them out): the fp32 and float64 decisions may differ there."""
    t, _ = view_space(scene, cam)
    radii = pre["radii"].copy()
    for k, tan in ((0, math.tan(cam.FoVx * 0.5)), (1, math.tan(cam.FoVy * 0.5))):
        lim = 1.3 * tan
        radii[np.abs(np.abs(t[:, k] / t[:, 2]) - lim) <= 1e-5 * lim] = 0
    return radii


CASES = [(3, True, False, "", False, 1), (2, True, True, "", False, 2), (1, True, False, "x", False, 3),
         (0, True, True, "xy", False, 4), (3, True, True, "y", True, 5), (0, False, True, "", True, 6),
         (0, False, False, "xy", False, 7)]


@pytest.mark.parametrize("deg,use_sh,depth,clamp,near,seed", CASES)
def test_host_camera_terms_match_float64(host_lib, deg, use_sh, depth, clamp, near, seed):
    scene, cam, pre, W, H = _scene(seed, deg, clamp, near)
    P = scene.P
    rng = np.random.default_rng(seed)
    g2d = rng.standard_normal((P, 3)).astype(np.float32)
    gconic = rng.standard_normal((P, 4)).astype(np.float32)
    gcol = rng.standard_normal((P, 3)).astype(np.float32)
    gz = rng.standard_normal((P, 1)).astype(np.float32) if depth else None
    radii = _drop_fragile(pre, scene, cam).astype(np.int32)
    cd = orc.cam_dict(cam)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    view, proj, cpos = f32(cd["viewmatrix"]).reshape(-1), f32(cd["projmatrix"]).reshape(-1), f32(cd["campos"]).reshape(-1)
    fx = np.float32(W) / (np.float32(2.0) * np.float32(cd["tanfovx"]))
    fy = np.float32(H) / (np.float32(2.0) * np.float32(cd["tanfovy"]))
    shs = f32(scene.shs) if use_sh else None
    M = shs.shape[1] if use_sh else 0
    clamped = np.ascontiguousarray(pre["clamped"], np.uint8)
    xyz, cov = f32(scene.xyz), f32(pre["cov3D"])
    out = np.zeros((P, 35), np.float32)
    scratch = np.zeros((16, 3), np.float32)
    host_lib.host_camera_grad(C.c_int(P), C.c_int(deg), C.c_int(M), _p(xyz), _p(radii), _p(shs), _p(clamped), _p(cov),
                              _p(view), _p(proj), C.c_float(fx), C.c_float(fy), C.c_float(cd["tanfovx"]),
                              C.c_float(cd["tanfovy"]), _p(cpos), _p(g2d), _p(gconic), _p(gcol),
                              _p(None if gz is None else f32(gz)), _p(scratch), _p(out))
    contrib, mag = camera_ref.camera_terms(xyz, radii, cov, view, proj, cpos, W, H, cd["tanfovx"], cd["tanfovy"], g2d,
                                           gconic, shs=shs, D=deg, clamped=clamped, dL_dcolors=gcol, dL_ddepth=gz)
    vis = radii > 0
    assert vis.sum() > 500
    assert not out[~vis].any()                                  # culled Gaussians contribute nothing
    for k in list(camera_ref.NEVER_READ_VIEW) + [16 + j for j in camera_ref.NEVER_READ_PROJ]:
        assert np.all(out[:, k] == 0), k                         # never-read entries are exactly 0, per Gaussian
    if not use_sh:
        assert not out[:, 32:].any()
    # the per-view sum, accumulated in float64 as the kernel does; the largest ratio measured here is 0.05 RTOL
    r = camera_ref.check_sum(out.astype(np.float64).sum(0), contrib, mag)
    assert r <= 1.0, r
    if clamp:
        t, _ = view_space(scene, cam)
        hit = vis & (np.abs(t[:, 0] / t[:, 2]) > 1.3 * math.tan(cam.FoVx * 0.5))
        hit |= vis & (np.abs(t[:, 1] / t[:, 2]) > 1.3 * math.tan(cam.FoVy * 0.5))
        assert hit.sum() > 5, "no clamped Gaussian survived the cull: the case is not exercised"
        sel = torch.as_tensor(hit)
        assert camera_ref.check_sum(out[hit].astype(np.float64).sum(0), contrib[sel], mag[sel]) <= 1.0
    if near:
        t, _ = view_space(scene, cam)
        hit = vis & (t[:, 2] < 0.36)
        assert hit.sum() > 5
        sel = torch.as_tensor(hit)
        assert camera_ref.check_sum(out[hit].astype(np.float64).sum(0), contrib[sel], mag[sel]) <= 1.0


def test_restatement_rejects_a_wrong_term(host_lib):
    """The comparison has teeth: the float64 sums with one Gaussian's view-gradient row dropped fail it."""
    scene, cam, pre, W, H = _scene(1, 3, "", False)
    P = scene.P
    rng = np.random.default_rng(0)
    g2d, gconic, gcol = (rng.standard_normal((P, k)).astype(np.float32) for k in (3, 4, 3))
    radii = _drop_fragile(pre, scene, cam).astype(np.int32)
    cd = orc.cam_dict(cam)
    contrib, mag = camera_ref.camera_terms(scene.xyz, radii, pre["cov3D"], cd["viewmatrix"], cd["projmatrix"],
                                           cd["campos"], W, H, cd["tanfovx"], cd["tanfovy"], g2d, gconic,
                                           shs=scene.shs, D=3, clamped=pre["clamped"], dL_dcolors=gcol)
    good = contrib.sum(0)
    assert camera_ref.check_sum(good, contrib, mag) == 0.0
    i = int(torch.argmax(contrib[:, 0].abs()))
    assert camera_ref.check_sum(good - contrib[i], contrib, mag) > 1.0
    bad = good.clone()
    bad[3] = 1e-30                                                 # a never-read entry must be exactly 0
    assert camera_ref.check_sum(bad, contrib, mag) == float("inf")


# ---------------------------------------------------------------- C ABI: argument rules of the _cam calls
def _inputs():
    return _lib.ViewInputs(P=10, D=0, M=0, W=64, H=64, C=3, background=1, means3D=1, shs=None, colors_precomp=1,
                           opacities=1, scales=1, scale_modifier=1.0, rotations=1, cov3D_precomp=None, viewmatrix=1,
                           projmatrix=1, campos=1, tan_fovx=0.5, tan_fovy=0.5, prefiltered=0, debug=0)


def _call(joint, cam_grads, V=2):
    lib = _lib.load()
    inp = _inputs()
    cams = (_lib.Camera * V)(*[_lib.Camera(1, 1, 1, 0.5, 0.5) for _ in range(V)])
    arr = (C.c_void_p * V)(*[1] * V)
    R = (C.c_int64 * V)(*[1] * V)
    grads = (_lib.ViewGrads * V)(*[_lib.ViewGrads(*[1] * 9) for _ in range(V)])
    cg = (_lib.CameraGrads * V)(*[_lib.CameraGrads(*t) for t in cam_grads])
    if joint:
        return lib.sgb_backward_joint_batch_cam(1, C.byref(inp), V, cams, R, arr, arr, arr, arr, arr, None, None,
                                                grads, 1, 8, 1, arr, 1, cg, None)
    return lib.sgb_backward_batch_cam(1, C.byref(inp), V, cams, R, arr, arr, arr, arr, arr, None, None, grads, cg,
                                      None)


@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("cam_grads,msg", [
    ([(100, 200, 300), (400, None, 600)], b"null camera-gradient output of view 1"),
    ([(None, 200, 300), (400, 500, 600)], b"null camera-gradient output of view 0"),
    ([(100, 200, 300), (400, 500, 100)], b"given twice"),
    ([(100, 100, 300), (400, 500, 600)], b"given twice"),
])
def test_bad_camera_grads_rejected_before_cuda(joint, cam_grads, msg):
    """Each bad argument returns SGB_E_INVALID during argument checking: no ctx is dereferenced and no CUDA call is
    made (the pointers are placeholders), so this runs without a GPU."""
    lib = _lib.load()
    assert _call(joint, cam_grads) == -1
    assert msg in lib.sgb_last_error()


def test_existing_rules_still_apply_to_cam_calls():
    lib = _lib.load()
    V = 2
    inp = _inputs()
    inp.C = 0
    cams = (_lib.Camera * V)(*[_lib.Camera(1, 1, 1, 0.5, 0.5) for _ in range(V)])
    arr = (C.c_void_p * V)(*[1] * V)
    R = (C.c_int64 * V)(*[1] * V)
    grads = (_lib.ViewGrads * V)(*[_lib.ViewGrads(*[1] * 9) for _ in range(V)])
    cg = (_lib.CameraGrads * V)(*[_lib.CameraGrads(1, 2, 3), _lib.CameraGrads(4, 5, 6)])
    assert lib.sgb_backward_batch_cam(1, C.byref(inp), V, cams, R, arr, arr, arr, arr, arr, None, None, grads, cg,
                                      None) == -1
    assert b"invalid sizes" in lib.sgb_last_error()


def test_cam_symbols_exported():
    lib = _lib.load()
    for name in ("sgb_backward_batch_cam", "sgb_backward_joint_batch_cam"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


# ---------------------------------------------------------------- pose correction module
class _Cam:
    pass


def _torch_cam(c, dtype=torch.float32):
    v = _Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
    v.world_view_transform = torch.as_tensor(c.world_view_transform).to(dtype)
    v.projection_matrix = torch.as_tensor(c.projection_matrix).to(dtype)
    v.full_proj_transform = torch.as_tensor(c.full_proj_transform).to(dtype)
    v.camera_center = torch.as_tensor(c.camera_center).to(dtype)
    v.uid, v.original_image = 17, torch.ones(3, 4, 5)
    return v


def test_rotation_matches_scipy():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(0)
    for scale in (0.0, 1e-9, 1e-4, 0.05, 0.0999, 0.1001, 0.5, 2.0, 3.1):
        for _ in range(4):
            w = rng.standard_normal(3)
            w = w / np.linalg.norm(w) * scale
            got = rotation(torch.as_tensor(w, dtype=torch.float64)).numpy()
            want = Rotation.from_rotvec(w).as_matrix()
            assert np.abs(got - want).max() <= 1e-15, (scale, np.abs(got - want).max())


def test_rotation_gradient_finite_at_zero():
    w = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    R = rotation(w)
    for i in range(3):
        for j in range(3):
            (g,) = torch.autograd.grad(R[i, j], w, retain_graph=True)
            assert torch.isfinite(g).all()
            # d R / d w_k at 0 is the generator [e_k]x
            want = torch.zeros(3, dtype=torch.float64)
            for k in range(3):
                e = torch.zeros(3, dtype=torch.float64)
                e[k] = 1.0
                want[k] = torch.linalg.cross(e, torch.eye(3, dtype=torch.float64)[j])[i]
            assert torch.equal(g, want)


def test_identity_at_zero_is_bitwise():
    cams = orbit_cameras(3, 64, 48)
    pose = CameraPoseCorrection(3, device="cpu")
    for i, c in enumerate(cams):
        cam = _torch_cam(c)
        cam.world_view_transform[0, 3] = -0.0           # a signed zero survives
        out = pose(cam, i)
        for name in ("world_view_transform", "full_proj_transform", "camera_center"):
            a, b = getattr(out, name), getattr(cam, name)
            assert a.dtype == b.dtype and a.shape == b.shape
            assert torch.equal(a.view(torch.int32), b.contiguous().view(torch.int32)), name


def test_delegates_other_attributes_and_builds_projection():
    c = orbit_cameras(1, 64, 48)[0]
    cam = _torch_cam(c)
    out = CameraPoseCorrection(1)(cam, 0)
    assert out.uid == 17 and out.image_width == 64 and out.FoVx == c.FoVx and out.original_image is cam.original_image
    del cam.projection_matrix
    out = CameraPoseCorrection(1)(cam, 0)
    assert torch.equal(out.projection_matrix, torch.as_tensor(c.projection_matrix))   # znear 0.01, zfar 100
    with pytest.raises(AttributeError):
        out.no_such_attribute


def _functional(out, wts):
    return sum((w * getattr(out, n)).sum() for n, w in zip(("world_view_transform", "full_proj_transform",
                                                            "camera_center"), wts))


def test_gradient_at_zero_matches_float64():
    c = orbit_cameras(2, 64, 48)[1]
    gen = torch.Generator().manual_seed(0)
    wts = [torch.randn(4, 4, generator=gen, dtype=torch.float64), torch.randn(4, 4, generator=gen, dtype=torch.float64),
           torch.randn(3, generator=gen, dtype=torch.float64)]
    p32 = CameraPoseCorrection(2)
    _functional(p32(_torch_cam(c), 1), [w.float() for w in wts]).backward()
    p64 = CameraPoseCorrection(2).double()
    _functional(p64(_torch_cam(c, torch.float64), 1), wts).backward()
    g32, g64 = p32.delta.grad[1].double(), p64.delta.grad[1]
    assert torch.isfinite(g32).all() and not p32.delta.grad[0].any()
    assert (g32 - g64).abs().max() <= 1e-5 * g64.abs().max()


def test_camera_center_is_inverse_of_view():
    c = orbit_cameras(2, 64, 48)[0]
    pose = CameraPoseCorrection(2)
    with torch.no_grad():
        pose.delta[0] = torch.tensor([0.02, -0.01, 0.015, 0.03, -0.02, 0.01])
        pose.delta[1] = torch.tensor([0.6, 0.3, -0.8, 0.5, 0.2, -0.4])
    for i in range(2):
        out = pose(_torch_cam(c), i)
        wvt = out.world_view_transform.double()
        want = torch.linalg.inv(wvt)[3, :3]
        got = out.camera_center.double()
        assert (got - want).abs().max() <= 8 * 2.0 ** -24 * (1 + want.abs().max()), (got, want)
        # full_proj_transform is world_view_transform' @ projection_matrix
        fp = (wvt @ out.projection_matrix.double())
        assert (out.full_proj_transform.double() - fp).abs().max() <= 8 * 2.0 ** -24 * fp.abs().max()
        # the motion acts in the camera frame: p_cam' = R p_cam + tau
        p = torch.tensor([0.3, -0.2, 0.5, 1.0], dtype=torch.float64)
        pc = p @ torch.as_tensor(c.world_view_transform).double()
        pc2 = p @ wvt
        d = pose.delta[i].detach().double()
        want_pc = rotation(d[:3]) @ pc[:3] + d[3:]
        assert (pc2[:3] - want_pc).abs().max() <= 1e-6
