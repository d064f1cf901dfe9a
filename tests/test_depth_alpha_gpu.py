"""Differentiable expected depth E = sum_i w_i z_i and accumulated opacity A = sum_i w_i of the RGB-D pass
(render_with_depth / render_batch(..., differentiable_depth=True)).

  * forward: E and A are bit for bit channels 0 and 1 of the same blend with features [depths, 1, 0] over
    background 0, and nothing the plain call returns moves;
  * backward: torch autograd through the plain render plus a second C = 3 render whose colours [z(means3D), 1, 0]
    are computed in torch is the reference; the blend-stage partials are checked against tests/blend_ref.py;
  * batch = per-view calls, no host synchronisation in the backward, and a short depth fit converges."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blend_ref as br  # noqa: E402
from raster_check import read_state  # noqa: E402
from util import frac_bad  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200 import channel_rasterization as chn  # noqa: E402
from semantic_gaussians_b200 import rgbd_rasterization as rgbd  # noqa: E402
from semantic_gaussians_b200 import rasterizer  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.renderer import _prepare, render, render_batch, render_with_depth  # noqa: E402
from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras  # noqa: E402

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


def _take_grads(leaves):
    out = [torch.zeros_like(t) if t.grad is None else t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    return out


_ROT = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]], np.float32)

# name: (P, W, H, sh degree, precomputed colours, pipe, world_rotate, scale_modifier, camera)
CASES = {
    "sh0": (20000, 160, 96, 0, False, Pipe, None, 1.0, "orbit"),
    "sh1": (20000, 160, 96, 1, False, Pipe, None, 1.0, "orbit"),
    "sh2": (20000, 160, 96, 2, False, Pipe, None, 1.0, "orbit"),
    "sh3": (20000, 160, 96, 3, False, Pipe, None, 1.0, "orbit"),
    "colors_precomp": (20000, 160, 96, 3, True, Pipe, None, 1.0, "orbit"),
    "cov3D_precomp": (20000, 160, 96, 3, False, CovPipe, None, 1.0, "orbit"),
    "world_rotate": (20000, 160, 96, 3, False, Pipe, _ROT, 1.0, "orbit"),
    "scale_modifier": (20000, 160, 96, 3, False, Pipe, None, 0.7, "orbit"),
    "ragged_333x211": (30000, 333, 211, 3, False, Pipe, None, 1.0, "orbit"),
    "all_culled": (20000, 160, 96, 3, False, Pipe, None, 1.0, "away"),
}


def _setup(name):
    P, W, H, deg, precomp, pipe, rot, mod, where = CASES[name]
    pc, leaves = _model(P, deg)
    c = orbit_cameras(4, W, H)[1] if where == "orbit" else look_at_camera((3.0, 0.0, 0.4), (6.0, 0.0, 0.4), W, H)
    colors = None
    if precomp:
        colors = torch.rand((P, 3), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
        colors.requires_grad_(True)
        leaves = leaves + [colors]
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    kw = dict(scaling_modifier=mod, override_color=colors, world_rotate=rot)
    return pc, leaves, _cam(c), pipe, bg, kw, (W, H)


def _depth_oracle_colors(cam, pc, pipe, kw, depths_from_state):
    """([z, 1, 0] colours of every Gaussian, the rasterizer call of render()): z either the kernel's own depth state
    (forward oracle) or restated in torch from means3D (backward oracle)."""
    pts, common, call = _prepare(cam, pc, pipe, kw["scaling_modifier"], kw["override_color"], None, None,
                                 kw["world_rotate"])
    if depths_from_state:
        args = (common["bg"] if "bg" in common else torch.zeros(3, device=DEV), call["means3D"],
                call["colors_precomp"] if call["colors_precomp"] is not None else torch.Tensor([]), call["opacities"],
                *[call[k] if call[k] is not None else torch.Tensor([]) for k in ("scales", "rotations")],
                common["scale_modifier"],
                call["cov3D_precomp"] if call["cov3D_precomp"] is not None else torch.Tensor([]),
                common["viewmatrix"], common["projmatrix"], common["tanfovx"], common["tanfovy"],
                common["image_height"], common["image_width"],
                call["shs"] if call["shs"] is not None else torch.Tensor([]), common["sh_degree"], common["campos"],
                False)
        with torch.no_grad():
            R, _, _, geom, binning, img, _ = rasterizer._C_rgbd.rasterize_gaussians(*args)
        P = call["means3D"].shape[0]
        z = read_state(_lib.load(), P, R, common["image_width"], common["image_height"], geom, binning, img,
                       ["depths"])["depths"]
    else:
        V = common["viewmatrix"].reshape(4, 4)
        z = call["means3D"] @ V[:3, 2] + V[3, 2]      # view-space z = V[2] x + V[6] y + V[10] z + V[14]
    return torch.stack([z, torch.ones_like(z), torch.zeros_like(z)], 1), pts, common, call


def _chn_render(common, call, means2D, colors):
    rs = chn.GaussianRasterizationSettings(bg=torch.zeros(3, device=DEV), debug=False, num_channels=3, **common)
    kw = {k: call[k] for k in ("means3D", "opacities", "scales", "rotations", "cov3D_precomp")}
    return chn.GaussianRasterizer(rs)(means2D=means2D, colors_precomp=colors, **kw)[0]


@pytest.mark.parametrize("name", list(CASES))
def test_forward_is_the_blend_of_depth_and_one_and_nothing_else_moves(name):
    pc, leaves, cam, pipe, bg, kw, (W, H) = _setup(name)
    with torch.no_grad():
        plain = render(cam, pc, pipe, bg, **kw)
        ours = render_with_depth(cam, pc, pipe, bg, **kw)
        feat, pts, common, call = _depth_oracle_colors(cam, pc, pipe, kw, True)
        oracle = _chn_render(common, call, pts, feat)
    assert set(ours) == set(plain) | {"expected_depth", "alpha"}
    for k in ("render", "depth", "radii", "visibility_filter"):
        assert torch.equal(ours[k], plain[k]), k
    assert ours["expected_depth"].shape == ours["alpha"].shape == (1, H, W)
    assert torch.equal(ours["expected_depth"][0], oracle[0])
    assert torch.equal(ours["alpha"][0], oracle[1])
    if name == "all_culled":
        assert not bool(plain["visibility_filter"].any()) and float(ours["alpha"].abs().max()) == 0.0
    else:
        assert float(ours["alpha"].max()) > 0.5


def test_forward_state_is_unchanged_by_the_option():
    """final_T and n_contrib of the image state, and every output, with the option on and off."""
    pc, _, cam, pipe, bg, kw, (W, H) = _setup("sh3")
    _, _, common, call = _depth_oracle_colors(cam, pc, pipe, kw, False)
    args = ([(common["viewmatrix"], common["projmatrix"], common["campos"], common["tanfovx"], common["tanfovy"])],
            bg, call["means3D"], None, call["opacities"], call["scales"], call["rotations"], 1.0, None, H, W,
            call["shs"], 3, False, False, 3)
    with torch.no_grad():
        runs = [rasterizer._forward(True, "t", *args, want_exp_alpha=on)[1] for on in (False, True)]
    lib, P = _lib.load(), call["means3D"].shape[0]
    states = [read_state(lib, P, r[0][0], W, H, r[3][0], r[4][0], r[5][0]) for r in runs]
    for k in ("final_T", "n_contrib", "point_list", "ranges"):
        assert torch.equal(states[0][k], states[1][k]), k
    for i in (1, 2, 6):   # colour, radii, median depth
        assert torch.equal(runs[0][i][0], runs[1][i][0])
    assert runs[0][7] is None and runs[1][7] is not None


@pytest.mark.parametrize("name", list(CASES))
def test_backward_matches_autograd_through_a_second_render(name):
    pc, leaves, cam, pipe, bg, kw, (W, H) = _setup(name)
    g = torch.Generator(device=DEV).manual_seed(11)
    dRGB, dE, dA = (torch.randn(s, device=DEV, generator=g) for s in ((3, H, W), (1, H, W), (1, H, W)))

    ours = render_with_depth(cam, pc, pipe, bg, **kw)
    ((ours["render"] * dRGB).sum() + (ours["expected_depth"] * dE).sum() + (ours["alpha"] * dA).sum()).backward()
    g_ours, vs_ours = _take_grads(leaves), ours["viewspace_points"].grad

    feat, pts, common, call = _depth_oracle_colors(cam, pc, pipe, kw, False)
    rs = rgbd.GaussianRasterizationSettings(bg=bg, debug=False, **common)
    rgb = rgbd.GaussianRasterizer(rs)(**call)[0]   # call["means2D"] is pts
    ch = _chn_render(common, call, pts, feat)
    ((rgb * dRGB).sum() + (ch[0] * dE[0]).sum() + (ch[1] * dA[0]).sum()).backward()
    g_ref, vs_ref = _take_grads(leaves), pts.grad

    for i, (a, b) in enumerate(zip(g_ours, g_ref)):
        assert frac_bad(a, b, rtol=1e-4, atol_scale=1e-4) == 0.0, i
    assert frac_bad(vs_ours, vs_ref, rtol=1e-4, atol_scale=1e-4) == 0.0
    if name != "all_culled":
        assert float(g_ours[0].abs().max()) > 0.0


def test_zero_depth_and_alpha_gradients_change_no_gradient():
    """Zero dL/dE and dL/dA through the extended backward give the plain backward's gradients.  Per-Gaussian sums
    are red.add reductions in scheduling order, so two runs of the same backward agree to re-association only; the
    comparison is at that run-to-run tolerance."""
    pc, leaves, cam, pipe, bg, kw, (W, H) = _setup("sh3")
    dRGB = torch.randn((3, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    plain = render(cam, pc, pipe, bg, **kw)
    (plain["render"] * dRGB).sum().backward()
    g_plain, vs_plain = _take_grads(leaves), plain["viewspace_points"].grad
    ours = render_with_depth(cam, pc, pipe, bg, **kw)
    ((ours["render"] * dRGB).sum() + (ours["expected_depth"] * 0).sum() + (ours["alpha"] * 0).sum()).backward()
    g_ours, vs_ours = _take_grads(leaves), ours["viewspace_points"].grad
    for a, b in zip(g_ours + [vs_ours], g_plain + [vs_plain]):
        assert frac_bad(a, b, rtol=1e-4, atol_scale=1e-5) == 0.0


def test_depth_only_loss_and_empty_scene():
    """A loss on E alone (no colour gradient) and P = 0 (zero planes, zero-size gradients)."""
    pc, leaves, cam, pipe, bg, kw, _ = _setup("sh3")
    out = render_with_depth(cam, pc, pipe, bg, **kw)
    out["expected_depth"].sum().backward()
    assert float(pc._xyz.grad.abs().max()) > 0.0 and float(pc._features_dc.grad.abs().max()) == 0.0

    W, H = 64, 48
    c = orbit_cameras(4, W, H)[1]
    z = lambda *s: torch.zeros(s, device=DEV, requires_grad=True)
    rs = rgbd.GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=math.tan(c.FoVx / 2), tanfovy=math.tan(c.FoVy / 2), bg=bg,
        scale_modifier=1.0, viewmatrix=torch.as_tensor(c.world_view_transform, device=DEV),
        projmatrix=torch.as_tensor(c.full_proj_transform, device=DEV), sh_degree=0,
        campos=torch.as_tensor(c.camera_center, device=DEV), prefiltered=False, debug=False)
    means3D, opac, cols = z(0, 3), z(0, 1), z(0, 3)
    color, radii, depth, E, A = rgbd.GaussianRasterizer(rs).forward_expected_depth(
        means3D=means3D, means2D=z(0, 3), opacities=opac, colors_precomp=cols, scales=z(0, 3), rotations=z(0, 4))
    assert E.shape == A.shape == (1, H, W) and float(E.abs().max()) == 0.0 and float(A.abs().max()) == 0.0
    (E.sum() + A.sum() + color.sum()).backward()
    assert means3D.grad.shape == (0, 3)


def test_blend_and_depth_gradients_match_fp64():
    """The extended backward with dL/dRGB = 0 on a colors_precomp scene, through the C ABI: dL/dmeans2D, dL/dconic and
    dL/dopacity against blend_ref.blend_backward on features [depths, 1] over background 0 (the kernel's own state),
    and dL/dmeans3D against geom_ref.geom_backward on the kernel's own blend gradients plus blend_ref's dL/dz
    (its dL/dfeature of the depth channel) times (V[2], V[6], V[10])."""
    import ctypes as Ct
    import geom_ref as gr
    W, H, P = 160, 96, 20000
    sc = make_scene(P, seed=21, scale_mean=0.03)
    c = orbit_cameras(4, W, H)[1]
    t = lambda a: torch.as_tensor(a, device=DEV).contiguous()
    means3D, scales, rots, opac = t(sc.xyz), t(sc.scales), t(sc.rotations), t(sc.opacity)
    colors = torch.rand((P, 3), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    view, proj, campos = t(c.world_view_transform), t(c.full_proj_transform), t(c.camera_center)
    tx, ty = math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    native, (R, _, radii, geom, binning, img, _, E, A) = rasterizer._forward(
        True, "t", [(view, proj, campos, tx, ty)], bg, means3D, colors, opac, scales, rots, 1.0, None, H, W, None, 0,
        False, False, 3, want_exp_alpha=True)
    lib = _lib.load()
    st = read_state(lib, P, R[0], W, H, geom[0], binning[0], img[0], ["depths", "cov3D"])
    feat = torch.stack([st["depths"], torch.ones_like(st["depths"])], 1)
    fargs = (st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], feat, torch.zeros(2), W, H)
    want_fwd = br.blend_forward(*fargs)
    assert br.compare(E[0][0], want_fwd["color"][0]) <= 1.0 and br.compare(A[0][0], want_fwd["color"][1]) <= 1.0
    dL = torch.randn((2, H * W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(9), dtype=torch.float64)
    dL[:, want_fwd["fragile"]] = 0.0
    dL = dL.float().reshape(2, 1, H, W).contiguous()
    z = lambda *s: torch.zeros(s, device=DEV)
    g = dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 4), dL_dopacity=z(P), dL_dcolors=z(P, 3), dL_dmeans3D=z(P, 3),
             dL_dcov3D=z(P, 6), dL_dsh=None, dL_dscales=z(P, 3), dL_drotations=z(P, 4))
    grads = _lib.ViewGrads(*[None if v is None else v.data_ptr() for v in g.values()])
    inp, cameras, _, _ = native
    vp = lambda x: Ct.c_void_p(x.data_ptr())
    stream, ctx = rasterizer._stream_ctx(DEV)
    dpix = z(3, H, W)
    _lib.check(lib.sgb_backward_batch_ext(ctx, Ct.byref(inp), 1, cameras, (Ct.c_int64 * 1)(R[0]), vp(radii[0]),
                                          vp(geom[0]), vp(binning[0]), vp(img[0]), vp(dpix), vp(dL[0]), vp(dL[1]),
                                          Ct.byref(grads), stream), "sgb_backward_batch_ext")
    want = br.blend_backward(*fargs, dL.reshape(2, H, W))
    errs = br.grad_errors({k: g[k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity")} | {"dL_dcolors": z(P, 2)},
                          dict(want, dL_dcolors=torch.zeros_like(want["dL_dcolors"])))
    camargs = (c.world_view_transform, c.full_proj_transform, c.camera_center, W, H, tx, ty)
    f = gr.geom_forward(means3D, opac, *camargs, scales=scales, rotations=rots)
    b = gr.geom_backward(means3D, radii[0], *camargs, st["cov3D"], g["dL_dmeans2D"], g["dL_dconic"], scales=scales,
                         rotations=rots)
    Vm = torch.as_tensor(c.world_view_transform, dtype=torch.float64, device=DEV).reshape(-1)
    dz = want["dL_dcolors"][:, 0:1].to(DEV) * Vm[[2, 6, 10]][None, :]
    want_m3 = gr.AV(b["dL_dmeans3D"].v + dz, b["dL_dmeans3D"].m + dz.abs())
    errs["dL_dmeans3D"] = gr.compare(g["dL_dmeans3D"], want_m3, ~f["fragile"])
    assert float(want_fwd["fragile"].double().mean()) <= 0.02
    assert float(dz.abs().max()) > 0.0
    assert all(e <= 1.0 for e in errs.values()), errs


def test_render_batch_equals_per_view_render():
    """Outputs bit for bit; gradients summed over the views equal the per-view sum up to the order of the fp32 sums
    (per-view buffers summed by torch against autograd accumulation), as for the plain batch path."""
    pc, leaves, _, pipe, bg, kw, (W, H) = _setup("sh3")
    cams = [_cam(c) for c in orbit_cameras(3, W, H)]
    gen = torch.Generator(device=DEV).manual_seed(6)
    dLs = [[torch.randn(s, device=DEV, generator=gen) for s in ((3, H, W), (1, H, W), (1, H, W))] for _ in cams]
    loss = lambda o, d: (o["render"] * d[0]).sum() + (o["expected_depth"] * d[1]).sum() + (o["alpha"] * d[2]).sum()
    single = [render_with_depth(c, pc, pipe, bg, **kw) for c in cams]
    sum(loss(o, d) for o, d in zip(single, dLs)).backward()
    g_single = _take_grads(leaves)
    batch = render_batch(cams, pc, pipe, bg, differentiable_depth=True, **kw)
    for o, b in zip(single, batch):
        assert set(o) == set(b)
        for k in ("render", "depth", "radii", "expected_depth", "alpha"):
            assert torch.equal(o[k], b[k]), k
    sum(loss(o, d) for o, d in zip(batch, dLs)).backward()
    for a, b in zip(_take_grads(leaves), g_single):
        assert frac_bad(a, b, rtol=1e-4, atol_scale=1e-4) == 0.0
    for o, b in zip(single, batch):
        assert frac_bad(b["viewspace_points"].grad, o["viewspace_points"].grad, rtol=1e-4, atol_scale=1e-4) == 0.0
    assert "expected_depth" not in render_batch(cams, pc, pipe, bg, **kw)[0]


def test_backward_adds_no_host_synchronisation():
    """The backward with the option on returns while the stream is still busy with work enqueued before it."""
    pc, leaves, cam, pipe, bg, kw, (W, H) = _setup("sh3")
    for warm in (True, False):   # the first backward sizes the ctx's dL/dz scratch
        out = render_with_depth(cam, pc, pipe, bg, **kw)
        loss = out["render"].sum() + out["expected_depth"].sum() + out["alpha"].sum()
        torch.cuda.synchronize()
        if not warm:
            torch.cuda._sleep(2_000_000_000)   # about a second of GPU clock cycles
        loss.backward()
        done = torch.cuda.Event()
        done.record()
        if not warm:
            assert not done.query(), "the backward waited for the GPU"
        torch.cuda.synchronize()
    assert float(pc._xyz.grad.abs().max()) > 0.0


def test_depth_fit_recovers_perturbed_positions():
    """Perturb every Gaussian's z, then 50 Adam steps on xyz with an L1 between the normalised expected depth
    E / max(A, eps) and that of the unperturbed scene (4 views, batched): the depth error over the covered pixels
    must fall below a quarter of its initial value (on an H100 it falls about twelvefold)."""
    W, H = 160, 120
    pc, _ = _model(20000, 3, seed=31, scale_mean=0.04)
    for t in (pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest):
        t.requires_grad_(False)
    cams = [_cam(c) for c in orbit_cameras(4, W, H)]
    bg = torch.zeros(3, device=DEV)

    def depth(outs):
        return [(o["expected_depth"] / o["alpha"].clamp_min(1e-4), o["alpha"]) for o in outs]

    with torch.no_grad():
        target = depth(render_batch(cams, pc, Pipe, bg, differentiable_depth=True))
        masks = [a > 0.5 for _, a in target]
        pc._xyz[:, 2] += 0.05 * torch.randn(pc._xyz.shape[0], device=DEV,
                                            generator=torch.Generator(device=DEV).manual_seed(8))

    def error(outs):
        return sum(float((d - t)[m].abs().mean()) for (d, _), (t, _), m in zip(depth(outs), target, masks)) / len(cams)

    opt = torch.optim.Adam([pc._xyz], lr=2e-3)
    with torch.no_grad():
        e0 = error(render_batch(cams, pc, Pipe, bg, differentiable_depth=True))
    for _ in range(50):
        outs = render_batch(cams, pc, Pipe, bg, differentiable_depth=True)
        loss = sum((d - t)[m].abs().mean() for (d, _), (t, _), m in zip(depth(outs), target, masks))
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        e1 = error(render_batch(cams, pc, Pipe, bg, differentiable_depth=True))
    print(f"\n[depth fit] mean |depth error| over covered pixels: {e0:.5f} -> {e1:.5f}")
    assert e1 < 0.25 * e0, (e0, e1)
