"""Anti-aliasing without a GPU: the geom_grad.cuh terms compiled for the host (tests/host/antialias_host.cpp) against
the float64 restatement (tests/antialias_ref.py) and float64 central differences, the C field's layout and argument
check, and the Python plumbing of the flag."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import antialias_ref as ar  # noqa: E402
from scene_recipes import push_sideways  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
U = 2.0 ** -24


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("aa") / "libaa_host.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++",
                           "-I", os.path.join(ROOT, "semantic-gaussians_b200", "csrc"),
                           os.path.join(HERE, "host", "antialias_host.cpp"), "-o", out])
    lib = C.CDLL(out)
    for f in ("host_aa_scale", "host_aa_cov_grad", "host_project_grad_aa"):
        getattr(lib, f).restype = None
    lib.host_project_grad_aa.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_float] * 4 + [C.c_void_p] * 5
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f32(*a):
    return [np.ascontiguousarray(x, np.float32) for x in a]


def _covs(kind, n=4000, seed=0):
    """Screen covariances C0 = (a0, b, c0) in px^2 of one family."""
    rng = np.random.default_rng(seed)
    if kind == "random":         # sub-pixel to tens of pixels, any orientation
        lam = 10 ** rng.uniform(-3, 2, (n, 2))
    elif kind == "anisotropic":  # needles: axis ratios up to 10^4
        lam = np.stack([10 ** rng.uniform(-4, -2, n), 10 ** rng.uniform(0, 2, n)], 1)
    elif kind == "near_singular":  # det C0 around eps * det C: both sides of the floor, and det C0 rounding negative
        lam = np.stack([10 ** rng.uniform(-7, -4.5, n), 10 ** rng.uniform(-1, 1, n)], 1)
    else:                        # b = 0: axis-aligned
        lam = 10 ** rng.uniform(-3, 2, (n, 2))
    th = rng.uniform(0, np.pi, n) if kind != "b0" else np.zeros(n)
    c, s = np.cos(th), np.sin(th)
    a0 = c * c * lam[:, 0] + s * s * lam[:, 1]
    b = c * s * (lam[:, 0] - lam[:, 1])
    c0 = s * s * lam[:, 0] + c * c * lam[:, 1]
    return _f32(a0, b, c0)


@pytest.mark.parametrize("kind", ["random", "anisotropic", "near_singular", "b0"])
def test_scale_matches_float64(host_lib, kind):
    a0, b, c0 = _covs(kind)
    n = a0.size
    hs = np.zeros(n, np.float32)
    host_lib.host_aa_scale(n, _p(a0), _p(b), _p(c0), _p(hs))
    r, h, active = ar.h_of(a0, b, c0)    # float64 on the fp32 inputs
    if kind == "near_singular":
        assert 0.1 < active.mean() < 0.9, active.mean()   # both branches reached
    D = (a0.astype(np.float64) + 0.3) * (c0 + 0.3) - b.astype(np.float64) ** 2
    # fp32 det C0 cancels: its error is a few ulps of a0 c0 + b^2, not of det C0
    tol_r = 8 * U * (np.abs(a0 * c0.astype(np.float64)) + b.astype(np.float64) ** 2) / D + 8 * U * np.abs(r)
    clear = np.abs(r - ar.EPS) > tol_r     # the branch is decided the same way away from the floor
    assert clear.mean() > 0.95
    assert ((hs > 0) == active)[clear].all()
    got = np.abs(hs).astype(np.float64)
    err = np.abs(got ** 2 - np.maximum(ar.EPS, r))
    assert (err <= tol_r + 8 * U * np.maximum(ar.EPS, r))[clear].all(), err.max()


@pytest.mark.parametrize("kind", ["random", "anisotropic", "near_singular", "b0"])
def test_cov_grad_matches_float64_and_central_differences(host_lib, kind):
    a0, b, c0 = _covs(kind, seed=1)
    n = a0.size
    g_r = np.random.default_rng(2).standard_normal(n).astype(np.float32)
    out = np.zeros((n, 3), np.float32)
    host_lib.host_aa_cov_grad(n, _p(a0), _p(b), _p(c0), _p(g_r), _p(out))
    want = ar.dr_dcov(a0, b, c0) * g_r[:, None].astype(np.float64)
    mag = np.abs(want).max(1, keepdims=True)
    # fp32 det C (and 0.3f for 0.3) against float64: a few ulps, more where (a0 + s)(c0 + s) and b^2 cancel
    A, Cc, B = a0 + 0.3, c0 + 0.3, b.astype(np.float64)
    cancel = ((A * Cc + B * B) / (A * Cc - B * B))[:, None]
    assert (np.abs(out - want) <= 16 * U * cancel * mag + 1e-30).all()
    if kind == "b0":
        assert not out[:, 1].any()
    # the float64 formula against central differences of r itself
    x = np.stack([a0, b, c0], 1).astype(np.float64)
    fd = np.zeros_like(x)
    for k in range(3):
        step = 1e-6 * np.maximum(np.abs(x).max(1), 1e-3)
        xp, xm = x.copy(), x.copy()
        xp[:, k] += step
        xm[:, k] -= step
        fd[:, k] = (ar.h_of(*xp.T)[0] - ar.h_of(*xm.T)[0]) / (2 * step)
    an = ar.dr_dcov(*x.T)
    assert (np.abs(fd - an) <= 1e-5 * np.abs(an).max(1, keepdims=True) + 1e-12).all()


@pytest.mark.parametrize("family", ["subpixel", "anisotropic", "sideways"])
def test_project_grad_term_matches_float64(host_lib, family):
    """project_grad with aa_g_r minus project_grad with aa_g_r = 0 (same conic and centre gradients) is
    d(g_r r)/d(means3D, cov3D): the term folded into dL/dC with the off-diagonal halved, then the existing chain.
    Against float64 autograd of the restated r, and that against central differences."""
    W, H = 160, 112
    scene = make_scene(3000, seed=5, sh=False, scale_mean=0.004 if family == "subpixel" else 0.03)
    cam = orbit_cameras(4, W, H)[1]
    if family == "anisotropic":
        rng = np.random.default_rng(3)
        scene.scales[:] *= (10 ** rng.uniform(-1.5, 1.5, scene.scales.shape)).astype(np.float32)
    if family == "sideways":
        push_sideways(scene, cam, "xy", every=3)
    xyz = np.ascontiguousarray(scene.xyz, np.float32)
    cov6 = ar.cov6_from_factors(torch.as_tensor(scene.scales, dtype=torch.float64),
                                torch.as_tensor(scene.rotations, dtype=torch.float64)).numpy().astype(np.float32)
    view = np.ascontiguousarray(np.asarray(cam.world_view_transform, np.float32).reshape(-1))
    proj = np.ascontiguousarray(np.asarray(cam.full_proj_transform, np.float32).reshape(-1))
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    fx, fy = np.float32(W) / (np.float32(2) * np.float32(tx)), np.float32(H) / (np.float32(2) * np.float32(ty))
    t = xyz @ view.reshape(4, 4)[:3, :3] + view.reshape(4, 4)[3, :3]
    keep = t[:, 2] > 0.5
    xyz, cov6 = np.ascontiguousarray(xyz[keep]), np.ascontiguousarray(cov6[keep])
    n = len(xyz)
    rng = np.random.default_rng(4)
    g_conic = rng.standard_normal((n, 3)).astype(np.float32)
    g_ndc = rng.standard_normal((n, 2)).astype(np.float32)
    g_r = rng.standard_normal(n).astype(np.float32)

    def run(gr):
        m, c = np.zeros((n, 3), np.float32), np.zeros((n, 6), np.float32)
        host_lib.host_project_grad_aa(n, _p(xyz), _p(cov6), _p(view), _p(proj), fx, fy, tx, ty, _p(g_conic),
                                      _p(g_ndc), _p(gr), _p(m), _p(c))
        return m.astype(np.float64), c.astype(np.float64)

    m1, c1 = run(g_r)
    m0, c0 = run(np.zeros(n, np.float32))
    P = torch.tensor(xyz, dtype=torch.float64, requires_grad=True)
    S6 = torch.tensor(cov6, dtype=torch.float64, requires_grad=True)
    a0, b, cc = ar.screen_cov0(P, S6, view, W, H, tx, ty)
    r = ar.r_torch(a0, b, cc)
    (torch.as_tensor(g_r, dtype=torch.float64) * r).sum().backward()
    want_m, want_c = P.grad.numpy(), S6.grad.numpy()
    # the difference of two fp32 evaluations: error relative to the whole gradient, not to the term alone
    mag_m = np.maximum(np.abs(m1), np.abs(m0)).max(1, keepdims=True) + np.abs(want_m).max(1, keepdims=True)
    mag_c = np.maximum(np.abs(c1), np.abs(c0)).max(1, keepdims=True) + np.abs(want_c).max(1, keepdims=True)
    bad_m = np.abs(m1 - m0 - want_m) > 2e-4 * mag_m
    bad_c = np.abs(c1 - c0 - want_c) > 2e-4 * mag_c
    assert bad_m.any(1).mean() < 0.01 and bad_c.any(1).mean() < 0.01, (bad_m.any(1).mean(), bad_c.any(1).mean())
    assert np.abs(want_c).max() > 0
    # the float64 restatement against central differences in cov3D (a sample of Gaussians)
    sel = np.arange(0, n, max(1, n // 50))
    for k in range(6):
        d = torch.zeros_like(S6)
        step = 1e-7 * S6.detach().abs().max(1).values
        d[:, k] = step
        with torch.no_grad():
            fp = ar.r_torch(*ar.screen_cov0(P, S6 + d, view, W, H, tx, ty))
            fm = ar.r_torch(*ar.screen_cov0(P, S6 - d, view, W, H, tx, ty))
        fd = (torch.as_tensor(g_r, dtype=torch.float64) * (fp - fm) / (2 * step)).numpy()
        assert np.allclose(fd[sel], want_c[sel, k], rtol=1e-4, atol=1e-6 * np.abs(want_c[sel]).max())


def test_view_inputs_layout_matches_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "sgb200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu\\n", sizeof(sgb_view_inputs), offsetof(sgb_view_inputs, debug),\n'
                   '         offsetof(sgb_view_inputs, antialiasing));\n  return 0;\n}\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    size, debug, aa = map(int, subprocess.check_output([exe], text=True).split())
    assert C.sizeof(_lib.ViewInputs) == size
    assert _lib.ViewInputs.debug.offset == debug and _lib.ViewInputs.antialiasing.offset == aa == debug + 4
    assert _lib.ViewInputs().antialiasing == 0


def _inputs(**kw):
    base = dict(P=10, D=0, M=0, W=64, H=64, C=3, background=1, means3D=1, shs=None, colors_precomp=1, opacities=1,
                scales=1, scale_modifier=1.0, rotations=1, cov3D_precomp=None, viewmatrix=1, projmatrix=1, campos=1,
                tan_fovx=0.5, tan_fovy=0.5, prefiltered=0, debug=0)
    base.update(kw)
    return _lib.ViewInputs(**base)


@pytest.mark.parametrize("value", [2, -1])
def test_bad_antialiasing_value_is_refused_before_cuda(value):
    lib = _lib.load()
    R = C.c_int64(0)
    rc = lib.sgb_forward_geometry(None, C.byref(_inputs(antialiasing=value)), None, None, C.byref(R), None)
    assert rc == -1 and f"antialiasing must be 0 or 1, got {value}".encode() in lib.sgb_last_error()
    cams = _lib.Camera(1, 1, 1, 0.5, 0.5)
    maps = C.c_void_p(1)
    inp = _inputs(antialiasing=value, colors_precomp=None, background=None)
    rc = lib.sgb_lift_batch(1, C.byref(inp), 1, C.byref(cams), C.byref(maps), _lib.FEAT_F32, 1, 1, None)
    assert rc == -1 and b"antialiasing must be 0 or 1" in lib.sgb_last_error()


def test_make_inputs_takes_the_flag(monkeypatch):
    """_make_inputs is the one place ViewInputs is filled: the flag arrives from the keyword of GaussianRasterizer,
    rasterize_batch, rasterize_joint_batch and from pipe.antialiasing in the renderer, and the settings are the
    reference's.  The native calls are replaced by a recorder (no GPU)."""
    from semantic_gaussians_b200 import channel_rasterization as chn
    from semantic_gaussians_b200 import rasterizer, renderer
    from semantic_gaussians_b200 import rgbd_rasterization as rgbd
    seen = []

    class Stop(Exception):
        pass

    def fake_forward(want_depth, what, *args, antialiasing=False, **kw):
        seen.append(antialiasing)
        raise Stop

    monkeypatch.setattr(rasterizer, "_forward", fake_forward)
    z = torch.zeros
    rs = chn.GaussianRasterizationSettings(8, 8, 1.0, 1.0, z(3), 1.0, torch.eye(4), torch.eye(4), 0, z(3), False,
                                           False, 3)
    kw = dict(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), colors_precomp=z(1, 3), scales=z(1, 3),
              rotations=z(1, 4))
    for aa in (False, True):
        with pytest.raises(Stop):
            chn.GaussianRasterizer(rs, antialiasing=aa)(**kw)
        with pytest.raises(Stop):
            chn.GaussianRasterizer.rasterize_batch(kw["means3D"], [kw["means2D"]], kw["opacities"], [rs],
                                                   colors_precomp=kw["colors_precomp"], scales=kw["scales"],
                                                   rotations=kw["rotations"], antialiasing=aa)
        rrs = rgbd.GaussianRasterizationSettings(*rs[:-1])
        with pytest.raises(Stop):
            rasterizer.rasterize_joint_batch(kw["means3D"], [kw["means2D"]], kw["opacities"], [rrs], z(1, 4), z(4),
                                             colors_precomp=kw["colors_precomp"], scales=kw["scales"],
                                             rotations=kw["rotations"], antialiasing=aa)
    assert seen == [False] * 3 + [True] * 3
    assert chn.GaussianRasterizer(rs).antialiasing is False
    assert chn.GaussianRasterizationSettings._fields[-1] == "num_channels"
    assert "antialiasing" not in chn.GaussianRasterizationSettings._fields
    assert "antialiasing" not in rgbd.GaussianRasterizationSettings._fields

    class Pipe:
        debug = False

    assert renderer._antialiasing(Pipe()) is False
    Pipe.antialiasing = True
    assert renderer._antialiasing(Pipe()) is True
