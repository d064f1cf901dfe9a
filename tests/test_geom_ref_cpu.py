"""The float64 geometry restatement (tests/geom_ref.py) on the CPU:
  - against the fp32 oracle (oracle/raster_oracle.c, which states forward.cu / backward.cu line by line): integer
    outputs equal except on fragile Gaussians, every float entry within RTOL * magnitude;
  - against central finite differences of its own forward, in float64: the backward is a derivative, not only a
    transcription;
  - against the product's gradient algebra (csrc/geom_grad.cuh) compiled for the host, entry by entry;
  - and the comparison rejects plausible bugs: each mutation of the restatement's backward exceeds the tolerance
    against the host build by at least 100x in its worst entry."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import geom_ref as gr  # noqa: E402
from scene_recipes import push_sideways  # noqa: E402

from oracle import oracle as orc  # noqa: E402

from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

ROOT = os.path.dirname(HERE)
W, H = 160, 112

# name: (SH degree, scale_modifier, cov3D_precomp, sideways axes, seed)
CASES = {f"d{D}": (D, 1.0, False, "", 1 + D) for D in range(4)}
CASES.update({"mod0.6": (3, 0.6, False, "", 5), "mod1.7": (2, 1.7, False, "", 6),
              "cov3D_precomp": (3, 1.0, True, "", 7), "sideways": (3, 1.7, False, "x", 9),
              "sideways_xy": (1, 1.0, False, "xy", 10)})


def _case(name):
    D, mod, precomp, axes, seed = CASES[name]
    scene = make_scene(4000, seed=seed, sh=True, scale_mean=0.08)
    cam = orbit_cameras(4, W, H)[seed % 4]
    sel = push_sideways(scene, cam, axes) if axes else None
    cd = orc.cam_dict(cam)
    cov = None
    if precomp:   # a covariance the scale / rotation path would not produce: the rotation of a non-unit quaternion
        q = scene.rotations * np.linspace(0.5, 2.0, scene.P, dtype=np.float32)[:, None]
        f = gr.geom_forward(scene.xyz, scene.opacity, cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H,
                            cd["tanfovx"], cd["tanfovy"], scales=scene.scales, rotations=q)
        cov = f["cov3D"].v.numpy().astype(np.float32)
    pre = orc.preprocess(scene.xyz, None if precomp else scene.scales, None if precomp else scene.rotations,
                         scene.opacity, cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H, cd["tanfovx"],
                         cd["tanfovy"], shs=scene.shs, cov3D_precomp=cov, scale_modifier=mod, sh_degree=D)
    rng = np.random.default_rng(seed)
    ups = dict(g2d=rng.standard_normal((scene.P, 3)).astype(np.float32),
               gconic=rng.standard_normal((scene.P, 4)).astype(np.float32),
               gcol=rng.standard_normal((scene.P, 3)).astype(np.float32))
    return dict(scene=scene, cam=cam, cd=cd, D=D, mod=mod, cov=cov, pre=pre, ups=ups, sel=sel)


def _camargs(k):
    cd = k["cd"]
    return (cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H, cd["tanfovx"], cd["tanfovy"])


def _ref_forward(k):
    s = k["scene"]
    f = k["cov"] is None
    return gr.geom_forward(s.xyz, s.opacity, *_camargs(k), scales=s.scales if f else None,
                           rotations=s.rotations if f else None, scale_modifier=k["mod"], cov3D_precomp=k["cov"],
                           shs=s.shs, D=k["D"])


def _ref_backward(k, mutation=None):
    s, pre, u = k["scene"], k["pre"], k["ups"]
    f = k["cov"] is None
    return gr.geom_backward(s.xyz, pre["radii"], *_camargs(k), pre["cov3D"], u["g2d"], u["gconic"],
                            scales=s.scales if f else None, rotations=s.rotations if f else None,
                            scale_modifier=k["mod"], shs=s.shs, D=k["D"], clamped=pre["clamped"],
                            dL_dcolors=u["gcol"], mutation=mutation)


def _native_backward(fn, k):
    """orc_geom_backward or the host build of geom_grad.cuh (same argument list) on the oracle's forward state."""
    s, pre, u, cd = k["scene"], k["pre"], k["ups"], k["cd"]
    P, M = s.P, s.shs.shape[1]
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)  # noqa: E731
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    out = dict(dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dcov3D=np.zeros((P, 6), np.float32),
               dL_dsh=np.zeros((P, M, 3), np.float32), dL_dscales=np.zeros((P, 3), np.float32),
               dL_drotations=np.zeros((P, 4), np.float32))
    view, proj, cpos = (f32(cd[n]).reshape(-1) for n in ("viewmatrix", "projmatrix", "campos"))
    fx = np.float32(W) / (np.float32(2.0) * np.float32(cd["tanfovx"]))
    fy = np.float32(H) / (np.float32(2.0) * np.float32(cd["tanfovy"]))
    factors = k["cov"] is None
    args = [f32(s.xyz), pre["radii"], f32(s.shs), pre["clamped"], f32(s.scales) if factors else None,
            f32(s.rotations) if factors else None]
    fn.restype = None
    fn(C.c_int(P), C.c_int(k["D"]), C.c_int(M), *[p(a) for a in args], C.c_float(k["mod"]), p(f32(pre["cov3D"])),
       p(view), p(proj), C.c_float(fx), C.c_float(fy), C.c_float(cd["tanfovx"]), C.c_float(cd["tanfovy"]), p(cpos),
       p(u["g2d"]), p(u["gconic"]), p(out["dL_dmeans3D"]), p(u["gcol"]), p(out["dL_dcov3D"]), p(out["dL_dsh"]),
       p(out["dL_dscales"]), p(out["dL_drotations"]))
    if not factors:
        del out["dL_dscales"], out["dL_drotations"]
    return out


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("geomref") / "libgeomgrad_host.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++",
                           "-I", os.path.join(ROOT, "semantic-gaussians_b200", "csrc"),
                           os.path.join(HERE, "host", "geom_grad_host.cpp"), "-o", out])
    return C.CDLL(out)


FRAGILE_MAX = 0.02


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_oracle(name):
    k = _case(name)
    f, pre = _ref_forward(k), k["pre"]
    ok = ~f["fragile"]
    vis = ok & f["visible"]
    frag = float(f["fragile"][~f["near"]].double().mean())
    assert frag <= FRAGILE_MAX
    assert int(vis.sum()) > 2000
    t = lambda a: torch.as_tensor(np.asarray(a).astype(np.int64))  # noqa: E731
    assert torch.equal(t(pre["radii"])[ok], f["radii"][ok])
    assert torch.equal(t(pre["tiles_touched"])[ok], f["tiles_touched"][ok])
    assert torch.equal(t(pre["rect"])[vis], f["rect"][vis])
    assert torch.equal(t(pre["clamped"]).bool()[vis], f["clamped"][vis])
    e = dict(depth=gr.compare(pre["depths"], f["depth"], vis), means2D=gr.compare(pre["means2D"], f["means2D"], vis),
             conic=gr.compare(pre["conic_opacity"][:, :3], f["conic"], vis), rgb=gr.compare(pre["rgb"], f["rgb"], vis))
    if k["cov"] is None:
        e["cov3D"] = gr.compare(pre["cov3D"], f["cov3D"], ok & ~f["near"])
    b = _ref_backward(k)
    got = _native_backward(orc.lib().orc_geom_backward, k)
    for n, g in got.items():
        e[n] = gr.compare(g, b[n], ok)
    print(f"\n[geom_ref vs oracle] {name}: fragile={frag:.4%} " + " ".join(f"{n}={x:.3g}" for n, x in e.items()))
    assert all(x <= 1.0 for x in e.values()), e
    if k["sel"] is not None:   # the clamp branch is reached
        cam = gr._camera(*_camargs(k))
        _, passes, _ = gr._clamp_t(gr._view_point(cam["view"], [gr._exact(torch.as_tensor(k["scene"].xyz[:, j]),
                                                                           "cpu") for j in range(3)]), cam)
        out = ~(passes[0] & passes[1]) & vis
        assert int(out.sum()) >= 20


def test_host_build_matches_restatement(host_lib):
    """The product's algebra (geom_grad.cuh, compiled for the host) per entry, with no quantile allowance."""
    for name in CASES:
        k = _case(name)
        ok = ~_ref_forward(k)["fragile"]
        b = _ref_backward(k)
        got = _native_backward(host_lib.host_geom_backward, k)
        e = {n: gr.compare(g, b[n], ok) for n, g in got.items()}
        print(f"\n[geom_ref vs host geom_grad.cuh] {name}: " + " ".join(f"{n}={x:.3g}" for n, x in e.items()))
        assert all(x <= 1.0 for x in e.values()), (name, e)


# which outputs each mutation changes, and a case that reaches it
MUTATION_CASES = dict(no_clamp_mask=("sideways", "dL_dmeans3D"), conic_xy_not_halved=("d3", "dL_dcov3D"),
                      cov_offdiag_not_doubled=("d3", "dL_dcov3D"), scale_times_modifier=("mod0.6", "dL_dscales"),
                      quat_xyzw=("d3", "dL_drotations"), no_sh_direction=("d3", "dL_dmeans3D"),
                      clamped_not_zeroed=("d3", "dL_dsh"), y1_sign=("d1", "dL_dsh"))


def test_comparison_rejects_plausible_bugs(host_lib):
    factors = {}
    for mut, (name, out) in MUTATION_CASES.items():
        k = _case(name)
        ok = ~_ref_forward(k)["fragile"]
        got = _native_backward(host_lib.host_geom_backward, k)
        assert gr.compare(got[out], _ref_backward(k)[out], ok) <= 1.0
        factors[mut] = gr.compare(got[out], _ref_backward(k, mutation=mut)[out], ok)
    print("\n[geom_ref mutations] worst entry / tolerance: " + " ".join(f"{m}={x:.3g}" for m, x in factors.items()))
    assert set(factors) == set(gr.MUTATIONS)
    assert all(x >= 100 for x in factors.values()), factors


def test_backward_is_the_derivative_of_the_forward():
    """Central differences of geom_forward in float64, per Gaussian (every Gaussian's outputs depend on its own
    inputs only, so one coordinate of all Gaussians is perturbed at once), against geom_backward with the 1e-7 of
    backward.cu:200 switched off.  The loss of Gaussian i is
        gx K_xx + 2 gy K_xy + gz K_yy + <g2d, ndc> + <gcol, rgb>
    for the conic K = (K_xx, K_xy, K_yy): the blend hands the geometry stage HALF the off-diagonal gradient
    (dL_dconic.y), hence the 2.  The checks on the conventions:
      - dL_dcov3D[1, 2, 4] is the derivative w.r.t. the stored off-diagonal entry, which appears twice in the
        symmetric matrix: the reference's "doubled" gradient;
      - dL_dscales is the derivative w.r.t. the modified scale mod * scale: the difference quotient w.r.t. scale
        divided by mod;
      - the quaternion is used as given, so the difference quotient w.r.t. its raw components is dL_drotations.
    Gaussians near the frustum clamp, culled, fragile or with a clamped colour channel are left out: there the
    forward is not differentiable, or the reference's convention is not the derivative."""
    scene = make_scene(1500, seed=21, sh=True, scale_mean=0.08)
    scene.rotations *= np.linspace(0.6, 1.6, scene.P, dtype=np.float32)[:, None]   # not unit: used as given
    cam = orbit_cameras(4, W, H)[2]
    cd = orc.cam_dict(cam)
    camargs = (cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H, cd["tanfovx"], cd["tanfovy"])
    D, mod = 3, 1.3
    P = scene.P
    x0 = dict(means=torch.as_tensor(scene.xyz, dtype=torch.float64),
              scales=torch.as_tensor(scene.scales, dtype=torch.float64),
              rot=torch.as_tensor(scene.rotations, dtype=torch.float64),
              sh=torch.as_tensor(scene.shs, dtype=torch.float64))
    rng = np.random.default_rng(3)
    g2d, gconic, gcol = (torch.as_tensor(rng.standard_normal(s)) for s in ((P, 3), (P, 4), (P, 3)))

    def fwd(x, cov=None):
        return gr.geom_forward(x["means"], scene.opacity, *camargs, scales=None if cov is not None else x["scales"],
                               rotations=None if cov is not None else x["rot"], scale_modifier=mod,
                               cov3D_precomp=cov, shs=x["sh"], D=D)

    def loss(f):
        ndc = [(f["means2D"].v[:, j] + 0.5) * 2.0 / (W, H)[j] - 1.0 for j in range(2)]
        k = f["conic"].v
        return (gconic[:, 0] * k[:, 0] + 2.0 * gconic[:, 1] * k[:, 1] + gconic[:, 3] * k[:, 2]
                + g2d[:, 0] * ndc[0] + g2d[:, 1] * ndc[1] + (gcol * f["rgb"].v).sum(1))

    f0 = fwd(x0)
    cam_ = gr._camera(*camargs)
    t = gr._view_point(cam_["view"], [gr._exact(x0["means"][:, j], "cpu") for j in range(3)])
    ratio_ok = ((t[0].v / t[2].v).abs() < 0.99 * cam_["limx"]) & ((t[1].v / t[2].v).abs() < 0.99 * cam_["limy"])
    use = f0["visible"] & ~f0["fragile"] & ratio_ok & ~f0["clamped"].any(1)
    assert int(use.sum()) > 800
    cov = f0["cov3D"].v
    b = gr.geom_backward(x0["means"], f0["radii"], *camargs, cov, g2d, gconic, scales=x0["scales"], rotations=x0["rot"],
                         scale_modifier=mod, shs=x0["sh"], D=D, clamped=f0["clamped"], dL_dcolors=gcol,
                         det_reg=False)
    bc = gr.geom_backward(x0["means"], f0["radii"], *camargs, cov, g2d, gconic, shs=x0["sh"], D=D,
                          clamped=f0["clamped"], dL_dcolors=gcol, det_reg=False)

    def fd(key, shape, cov_input=False):
        out = torch.zeros((P,) + shape, dtype=torch.float64)
        for idx in np.ndindex(*shape):
            h = 1e-6
            xs = []
            for sgn in (1.0, -1.0):
                if cov_input:
                    c = cov.clone()
                    c[(slice(None),) + idx] += sgn * h
                    xs.append(loss(fwd(x0, c)))
                else:
                    x = dict(x0)
                    x[key] = x0[key].clone()
                    x[key][(slice(None),) + idx] += sgn * h
                    xs.append(loss(fwd(x)))
            out[(slice(None),) + idx] = (xs[0] - xs[1]) / (2 * h)
        return out

    n = (D + 1) ** 2
    checks = dict(dL_dmeans3D=(fd("means", (3,)), b["dL_dmeans3D"]),
                  dL_dscales=(fd("scales", (3,)) / gr._c(mod), b["dL_dscales"]),
                  dL_drotations=(fd("rot", (4,)), b["dL_drotations"]),
                  dL_dsh=(fd("sh", (n, 3)), b["dL_dsh"][:, :n]),
                  dL_dcov3D=(fd(None, (6,), cov_input=True), bc["dL_dcov3D"]))
    errs = {}
    for name, (num, want) in checks.items():
        # float64 central differences with h = 1e-6 are good to ~1e-8 of the terms' magnitude
        errs[name] = gr.compare(num, want, use, rtol=1e-6)
    print("\n[geom_ref vs finite differences] " + " ".join(f"{k}={x:.3g}" for k, x in errs.items()))
    assert all(x <= 1.0 for x in errs.values()), errs
