"""The anti-aliasing part of the float64 geometry restatement (tests/geom_ref.py, antialiasing=True) on the CPU:
  - against the independent autograd restatement of tests/antialias_ref.py (h, dL/do and the covariance term's chain
    to means3D, cov3D, scales and rotations) to about 1e-12 of the magnitude;
  - against central differences of geom_ref's own forward: the backward is the derivative of o h;
  - against the product's algebra (geom_grad.cuh, compiled for the host as geom_backward_kernel<false, true> runs it,
    tests/host/antialias_host.cpp), entry by entry within geom_ref.RTOL * magnitude;
  - and every anti-aliasing mutation of the restatement's backward exceeds that tolerance against the host build by
    at least 100x in its worst entry."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import antialias_ref as ar  # noqa: E402
import geom_ref as gr  # noqa: E402
from scene_recipes import push_sideways  # noqa: E402

from oracle import oracle as orc  # noqa: E402

from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

ROOT = os.path.dirname(HERE)
W, H = 160, 112
FRAGILE_MAX = 0.02

# name: (SH degree, scale_modifier, cov3D_precomp, sideways axes, seed, family)
CASES = {"d3": (3, 1.0, False, "", 2, None), "d1_mod1.7": (1, 1.7, False, "", 6, None),
         "cov3D_precomp": (3, 1.0, True, "", 7, None), "sideways_xy": (1, 1.0, False, "xy", 10, None),
         "needles": (3, 1.0, False, "", 11, "needles"), "subpixel": (0, 0.6, False, "", 12, "subpixel")}


def _case(name):
    D, mod, precomp, axes, seed, family = CASES[name]
    scene = make_scene(4000, seed=seed, sh=True, scale_mean=0.08)
    cam = orbit_cameras(4, W, H)[seed % 4]
    i = np.arange(scene.P)
    rng = np.random.default_rng(seed)
    if family == "needles":      # det C0 cancels: a0 c0 close to b^2 (thinner ones make the floor decision fragile)
        n = int((i % 8 == 0).sum())
        scene.scales[i % 8 == 0] = np.array([0.3, 2e-3, 2e-3], np.float32) * rng.uniform(0.5, 2, (n, 1)).astype(np.float32)
    if family == "subpixel":     # det C0 / det C across the floor 2.5e-5
        scene.scales[i % 2 == 0] = (10 ** rng.uniform(-4.5, -2.5, (int((i % 2 == 0).sum()), 3))).astype(np.float32)
    sel = push_sideways(scene, cam, axes) if axes else None
    cd = orc.cam_dict(cam)
    cov = None
    if precomp:
        q = scene.rotations * np.linspace(0.5, 2.0, scene.P, dtype=np.float32)[:, None]
        f = gr.geom_forward(scene.xyz, scene.opacity, cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H,
                            cd["tanfovx"], cd["tanfovy"], scales=scene.scales, rotations=q)
        cov = f["cov3D"].v.numpy().astype(np.float32)
    pre = orc.preprocess(scene.xyz, None if precomp else scene.scales, None if precomp else scene.rotations,
                         scene.opacity, cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H, cd["tanfovx"],
                         cd["tanfovy"], shs=scene.shs, cov3D_precomp=cov, scale_modifier=mod, sh_degree=D)
    ups = dict(g2d=rng.standard_normal((scene.P, 3)).astype(np.float32),
               gconic=rng.standard_normal((scene.P, 4)).astype(np.float32),
               gcol=rng.standard_normal((scene.P, 3)).astype(np.float32),
               gop=rng.standard_normal(scene.P).astype(np.float32))
    ups["gop"][np.asarray(pre["radii"]).reshape(-1) <= 0] = 0.0     # the blend gives culled Gaussians nothing
    return dict(scene=scene, cam=cam, cd=cd, D=D, mod=mod, cov=cov, pre=pre, ups=ups, sel=sel, family=family)


def _camargs(k):
    cd = k["cd"]
    return (cd["viewmatrix"], cd["projmatrix"], cd["campos"], W, H, cd["tanfovx"], cd["tanfovy"])


def _ref_forward(k):
    s = k["scene"]
    f = k["cov"] is None
    return gr.geom_forward(s.xyz, s.opacity, *_camargs(k), scales=s.scales if f else None,
                           rotations=s.rotations if f else None, scale_modifier=k["mod"], cov3D_precomp=k["cov"],
                           shs=s.shs, D=k["D"], antialiasing=True)


def _ref_backward(k, mutation=None):
    s, pre, u = k["scene"], k["pre"], k["ups"]
    f = k["cov"] is None
    return gr.geom_backward(s.xyz, pre["radii"], *_camargs(k), pre["cov3D"], u["g2d"], u["gconic"],
                            scales=s.scales if f else None, rotations=s.rotations if f else None,
                            scale_modifier=k["mod"], shs=s.shs, D=k["D"], clamped=pre["clamped"],
                            dL_dcolors=u["gcol"], mutation=mutation, antialiasing=True, opacities=s.opacity,
                            dL_dopacity=u["gop"])


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("aaref") / "libaa_host.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-x", "c++",
                           "-I", os.path.join(ROOT, "semantic-gaussians_b200", "csrc"),
                           os.path.join(HERE, "host", "antialias_host.cpp"), "-o", out])
    lib = C.CDLL(out)
    lib.host_aa_scale.restype = None
    lib.host_geom_backward_aa.restype = None
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _host_h(lib, f):
    """The signed h the forward kernel stores, from fp32 (a0, b, c0) (host build of aa_scale)."""
    cov0 = np.ascontiguousarray(f["aa_cov0"].v.numpy().astype(np.float32).T)
    hs = np.zeros(cov0.shape[1], np.float32)
    lib.host_aa_scale(C.c_int(hs.size), *[_p(np.ascontiguousarray(x)) for x in cov0], _p(hs))
    return hs


def _host_backward(lib, k, hs):
    s, pre, u, cd = k["scene"], k["pre"], k["ups"], k["cd"]
    P, M = s.P, s.shs.shape[1]
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)  # noqa: E731
    out = dict(dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dcov3D=np.zeros((P, 6), np.float32),
               dL_dsh=np.zeros((P, M, 3), np.float32), dL_dscales=np.zeros((P, 3), np.float32),
               dL_drotations=np.zeros((P, 4), np.float32), dL_dopacity=f32(u["gop"]).copy())
    view, proj, cpos = (f32(cd[n]).reshape(-1) for n in ("viewmatrix", "projmatrix", "campos"))
    fx = np.float32(W) / (np.float32(2.0) * np.float32(cd["tanfovx"]))
    fy = np.float32(H) / (np.float32(2.0) * np.float32(cd["tanfovy"]))
    factors = k["cov"] is None
    args = [f32(s.xyz), pre["radii"], f32(s.shs), pre["clamped"], f32(s.scales) if factors else None,
            f32(s.rotations) if factors else None]
    lib.host_geom_backward_aa(C.c_int(P), C.c_int(k["D"]), C.c_int(M), *[_p(a) for a in args], C.c_float(k["mod"]),
                              _p(f32(pre["cov3D"])), _p(view), _p(proj), C.c_float(fx), C.c_float(fy),
                              C.c_float(cd["tanfovx"]), C.c_float(cd["tanfovy"]), _p(cpos), _p(u["g2d"]),
                              _p(u["gconic"]), _p(out["dL_dmeans3D"]), _p(u["gcol"]), _p(out["dL_dcov3D"]),
                              _p(out["dL_dsh"]), _p(out["dL_dscales"]), _p(out["dL_drotations"]),
                              _p(f32(s.opacity).reshape(-1)), _p(hs), _p(out["dL_dopacity"]))
    if not factors:
        del out["dL_dscales"], out["dL_drotations"]
    return out


def test_families_reach_the_anti_aliasing_branches():
    """needles: det C0 cancels (its conditioning kappa0 above 1e3); subpixel: r on both sides of the floor."""
    f = _ref_forward(_case("needles"))
    vis = f["visible"] & ~f["fragile"]
    a0, b, c0 = (f["aa_cov0"].v[:, j] for j in range(3))
    kappa0 = ((a0 * c0).abs() + b * b) / (a0 * c0 - b * b).abs()
    n = int((vis & f["aa_active"] & (kappa0 > 1e3)).sum())
    print(f"\nneedles: {n} above the floor with kappa0 > 1e3")
    assert n >= 100
    f = _ref_forward(_case("subpixel"))
    vis = f["visible"] & ~f["fragile"]
    print(f"\nsubpixel: {int((vis & f['aa_active']).sum())} above the floor, {int((vis & ~f['aa_active']).sum())} on it")
    assert int((vis & f["aa_active"]).sum()) >= 200 and int((vis & ~f["aa_active"]).sum()) >= 200


@pytest.mark.parametrize("name", ["d3", "needles", "subpixel", "cov3D_precomp"])
def test_restatement_matches_autograd(name, monkeypatch):
    """geom_ref's h and o h against antialias_ref.h_of, and its backward (with only the opacity gradient upstream,
    so that all of it is the anti-aliasing term) against float64 autograd of sum g o h through antialias_ref's
    screen covariance and covariance factorisation.  Focal lengths, the dilation and the floor are held at the fp32
    values the kernels use (0.3f and 2.5e-5f differ from 0.3 and 2.5e-5 by 4e-8 relative)."""
    monkeypatch.setattr(ar, "S", gr.AA_DILATION)
    monkeypatch.setattr(ar, "EPS", gr.AA_FLOOR)
    k = _case(name)
    s = k["scene"]
    f = _ref_forward(k)
    keep = f["visible"] & ~f["fragile"]
    cam = gr._camera(*_camargs(k))
    P = s.P
    view = np.asarray(k["cd"]["viewmatrix"], np.float32).reshape(-1)
    tx, ty = W / (2.0 * cam["fx"]), H / (2.0 * cam["fy"])         # W / (2 tx) is the fp32 focal length exactly
    pos = torch.tensor(s.xyz, dtype=torch.float64, requires_grad=True)
    if k["cov"] is None:
        sc = torch.tensor(s.scales, dtype=torch.float64, requires_grad=True)
        rot = torch.tensor(s.rotations, dtype=torch.float64, requires_grad=True)
        cov6 = ar.cov6_from_factors(sc, rot, gr._c(k["mod"]))
    else:
        cov6 = torch.tensor(k["cov"], dtype=torch.float64, requires_grad=True)
    a0, b, c0 = ar.screen_cov0(pos, cov6, view, W, H, tx, ty)
    t = gr._view_point(cam["view"], [gr._exact(torch.as_tensor(s.xyz[:, j]), "cpu") for j in range(3)])
    inside = ((t[0].v / t[2].v).abs() < 0.99 * cam["limx"]) & ((t[1].v / t[2].v).abs() < 0.99 * cam["limy"])
    keep &= inside    # the clamp limits are 1.3 tan in fp32 here, in float64 there
    r, h_want, active = ar.h_of(a0.detach().numpy(), b.detach().numpy(), c0.detach().numpy())
    assert np.array_equal(active[keep.numpy()], f["aa_active"][keep].numpy())
    e = {"h": gr.compare(torch.as_tensor(h_want), f["aa_h"], keep, rtol=1e-12)}
    g = torch.as_tensor(k["ups"]["gop"], dtype=torch.float64)
    o = torch.as_tensor(s.opacity, dtype=torch.float64).reshape(-1)
    e["aa_opacity"] = gr.compare(o * torch.as_tensor(h_want), f["aa_opacity"], keep, rtol=1e-12)
    rr = ar.r_torch(a0, b, c0)
    h_t = torch.where(torch.as_tensor(active), rr.clamp(min=ar.EPS).sqrt(), torch.full_like(rr, ar.EPS ** 0.5))
    (o * g * h_t * keep.double()).sum().backward()
    zero = np.zeros((P, 3), np.float32)
    bw = gr.geom_backward(s.xyz, k["pre"]["radii"], *_camargs(k), cov6.detach().numpy(), zero,
                          np.zeros((P, 4), np.float32), scales=s.scales if k["cov"] is None else None,
                          rotations=s.rotations if k["cov"] is None else None, scale_modifier=k["mod"],
                          det_reg=False, antialiasing=True, opacities=s.opacity, dL_dopacity=k["ups"]["gop"])
    e["dL_dopacity"] = gr.compare(torch.as_tensor(h_want) * g, bw["dL_dopacity"], keep, rtol=1e-12)
    e["dL_dmeans3D"] = gr.compare(pos.grad, bw["dL_dmeans3D"], keep, rtol=1e-12)
    if k["cov"] is None:
        e["dL_dscales"] = gr.compare(sc.grad / gr._c(k["mod"]), bw["dL_dscales"], keep, rtol=1e-12)
        e["dL_drotations"] = gr.compare(rot.grad, bw["dL_drotations"], keep, rtol=1e-12)
    else:
        e["dL_dcov3D"] = gr.compare(cov6.grad, bw["dL_dcov3D"], keep, rtol=1e-12)
    print(f"\n[geom_ref AA vs autograd] {name}: " + " ".join(f"{n}={x:.3g}" for n, x in e.items()))
    assert float(bw["dL_dmeans3D"].v[keep].abs().max()) > 0
    assert all(x <= 1.0 for x in e.values()), e


def test_backward_is_the_derivative_of_o_h():
    """Central differences of sum g o h(geom_forward) in float64 against geom_backward with only the opacity
    gradient upstream; Gaussians near the frustum clamp, near the floor (|r / eps - 1| < 1e-3) or fragile are left
    out."""
    k = _case("subpixel")
    s = k["scene"]
    s.rotations *= np.linspace(0.6, 1.6, s.P, dtype=np.float32)[:, None]
    camargs = _camargs(k)
    mod = gr._c(k["mod"])
    g = torch.as_tensor(k["ups"]["gop"], dtype=torch.float64)
    x0 = dict(means=torch.as_tensor(s.xyz, dtype=torch.float64), scales=torch.as_tensor(s.scales, dtype=torch.float64),
              rot=torch.as_tensor(s.rotations, dtype=torch.float64))

    def loss(x):
        f = gr.geom_forward(x["means"], s.opacity, *camargs, scales=x["scales"], rotations=x["rot"],
                            scale_modifier=k["mod"], antialiasing=True)
        return g * f["aa_opacity"].v

    f0 = gr.geom_forward(x0["means"], s.opacity, *camargs, scales=x0["scales"], rotations=x0["rot"],
                         scale_modifier=k["mod"], antialiasing=True)
    cam = gr._camera(*camargs)
    t = gr._view_point(cam["view"], [gr._exact(x0["means"][:, j], "cpu") for j in range(3)])
    ratio_ok = ((t[0].v / t[2].v).abs() < 0.99 * cam["limx"]) & ((t[1].v / t[2].v).abs() < 0.99 * cam["limy"])
    a0, b, c0 = (f0["aa_cov0"].v[:, j] for j in range(3))
    r = ar.r_torch(a0, b, c0)
    use = f0["visible"] & ~f0["fragile"] & ratio_ok & ((r / ar.EPS - 1).abs() > 1e-3)
    assert int((use & f0["aa_active"]).sum()) > 500 and int((use & ~f0["aa_active"]).sum()) > 200
    P = s.P
    bw = gr.geom_backward(x0["means"], f0["radii"], *camargs, f0["cov3D"].v, np.zeros((P, 3)), np.zeros((P, 4)),
                          scales=x0["scales"], rotations=x0["rot"], scale_modifier=k["mod"], det_reg=False,
                          antialiasing=True, opacities=s.opacity, dL_dopacity=g)

    def fd(key, n):
        out = torch.zeros((P, n), dtype=torch.float64)
        for j in range(n):
            vals = []
            for sgn in (1.0, -1.0):
                x = dict(x0)
                x[key] = x0[key].clone()
                x[key][:, j] += sgn * 1e-7 * x0[key][:, j].abs().clamp(min=1e-3)
                vals.append(loss(x))
            out[:, j] = (vals[0] - vals[1]) / (2e-7 * x0[key][:, j].abs().clamp(min=1e-3))
        return out

    errs = dict(dL_dmeans3D=gr.compare(fd("means", 3), bw["dL_dmeans3D"], use, rtol=1e-5),
                dL_dscales=gr.compare(fd("scales", 3) / mod, bw["dL_dscales"], use, rtol=1e-5),
                dL_drotations=gr.compare(fd("rot", 4), bw["dL_drotations"], use, rtol=1e-5))
    print("\n[geom_ref AA vs finite differences] " + " ".join(f"{n}={x:.3g}" for n, x in errs.items()))
    assert all(x <= 1.0 for x in errs.values()), errs
    floor = use & ~f0["aa_active"]
    assert float(bw["dL_dmeans3D"].v[floor].abs().max()) == 0.0     # nothing on the floor branch


@pytest.mark.parametrize("name", list(CASES))
def test_host_build_matches_restatement(host_lib, name):
    k = _case(name)
    f = _ref_forward(k)
    ok = ~f["fragile"]
    frag = float(f["fragile"][~f["near"]].double().mean())
    assert frag <= FRAGILE_MAX
    hs = _host_h(host_lib, f)
    vis = ok & f["visible"]
    e = {"aa_h": gr.compare(np.abs(hs), f["aa_h"], vis)}
    assert np.array_equal(hs[vis.numpy()] > 0, f["aa_active"][vis].numpy())
    b = _ref_backward(k)
    got = _host_backward(host_lib, k, hs)
    e.update({n: gr.compare(g, b[n], ok) for n, g in got.items()})
    print(f"\n[geom_ref AA vs host geom_grad.cuh] {name}: fragile={frag:.4%} " +
          " ".join(f"{n}={x:.3g}" for n, x in e.items()))
    assert all(x <= 1.0 for x in e.values()), e


# which output each anti-aliasing mutation changes, and a case that reaches it
MUTATION_CASES = dict(aa_offdiag_not_halved=("d3", "dL_dcov3D"), aa_cov_on_floor=("subpixel", "dL_dmeans3D"),
                      aa_dopacity_not_scaled=("d3", "dL_dopacity"), aa_det_swapped=("needles", "dL_dcov3D"),
                      aa_h_squared=("d3", "dL_dopacity"))


def test_comparison_rejects_anti_aliasing_bugs(host_lib):
    factors = {}
    for mut, (name, out) in MUTATION_CASES.items():
        k = _case(name)
        f = _ref_forward(k)
        ok = ~f["fragile"]
        got = _host_backward(host_lib, k, _host_h(host_lib, f))
        assert gr.compare(got[out], _ref_backward(k)[out], ok) <= 1.0
        factors[mut] = gr.compare(got[out], _ref_backward(k, mutation=mut)[out], ok)
    print("\n[geom_ref AA mutations] worst entry / tolerance: " + " ".join(f"{m}={x:.3g}" for m, x in factors.items()))
    assert set(factors) == set(gr.AA_MUTATIONS)
    assert all(x >= 100 for x in factors.values()), factors
