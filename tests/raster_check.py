"""The kernels of one forward + backward against the float64 restatements, through the C ABI: the blend
(tests/blend_ref.py) and the per-Gaussian geometry (tests/geom_ref.py).  Both restatements run on the kernels' own
state (sgb_state_field) and, in the backward, on the kernels' own upstream gradients, so the only error measured is
each stage's own arithmetic."""
import ctypes as Ct
import math
import time

import torch

import blend_ref as br
import geom_ref as gr
from util import dev_cam, dev_scene

from semantic_gaussians_b200 import _lib

FRAGILE_MAX = 0.02   # at most this fraction of pixels (blend) or Gaussians (geometry) may be left out
DEV = torch.device("cuda:0")


def read_state(lib, P, R, W, H, geom, binning, img, fields=None):
    """The blend's inputs and forward state of one view, as the kernels left them; `fields` adds per-Gaussian
    geometry fields ("depths", "cov3D", "rgb", "clamped", "tiles_touched")."""
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    spec = dict(means2D=(torch.float32, (P, 2)), conic_opacity=(torch.float32, (P, 4)),
                point_list=(torch.int32, (max(R, 1),)), ranges=(torch.int32, (tiles, 2)),
                n_contrib=(torch.int32, (H * W,)), final_T=(torch.float32, (H * W,)))
    extra = dict(depths=(torch.float32, (P,)), cov3D=(torch.float32, (P, 6)), rgb=(torch.float32, (P, 3)),
                 clamped=(torch.uint8, (P, 3)), tiles_touched=(torch.int32, (P,)))
    spec.update({k: extra[k] for k in (fields or ())})
    st = {}
    for name, (dt, shape) in spec.items():
        t = torch.zeros(shape, dtype=dt, device=DEV)
        n = lib.sgb_state_field(name.encode(), P, R, W, H, geom.data_ptr(), binning.data_ptr(), img.data_ptr(),
                                t.data_ptr(), torch.cuda.current_stream(DEV).cuda_stream)
        assert n >= 0, lib.sgb_last_error()
        st[name] = t[:R] if name == "point_list" else t
    return st


def _placed(t, offset):
    """A copy of t whose data pointer is `offset` bytes past a 16-byte boundary (the C ABI takes any pointer)."""
    buf = torch.zeros(t.numel() + 4, dtype=t.dtype, device=t.device)
    v = buf[offset // 4: offset // 4 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == offset
    return v


GEOM_GRADS = ("dL_dmeans3D", "dL_dcov3D", "dL_dscales", "dL_drotations", "dL_dsh")


def _geometry_errors(sc, cam, W, H, inp_args, st, radii, grads, dcolors_view):
    """Every forward geometry field and every geometry gradient of one view against geom_ref.  Returns
    (errors, fragile fraction, forward restatement)."""
    shs, D, mod, cov_pre = inp_args["shs"], inp_args["D"], inp_args["scale_modifier"], inp_args["cov3D_precomp"]
    factors = cov_pre is None
    camargs = (cam.world_view_transform, cam.full_proj_transform, cam.camera_center, W, H,
               math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5))
    f = gr.geom_forward(sc["means3D"], sc["opacities"], *camargs, scales=sc["scales"] if factors else None,
                        rotations=sc["rotations"] if factors else None, scale_modifier=mod, cov3D_precomp=cov_pre,
                        shs=shs, D=D)
    ok = ~f["fragile"]
    vis = f["visible"] & ok
    # integers: equal except on fragile Gaussians
    assert torch.equal(radii.long()[ok], f["radii"][ok])
    assert torch.equal(st["tiles_touched"].long()[ok], f["tiles_touched"][ok])
    if shs is not None:
        assert torch.equal(st["clamped"].bool()[vis], f["clamped"][vis])
    assert torch.equal(st["conic_opacity"][vis, 3], sc["opacities"].reshape(-1)[vis])
    e = {"depth": gr.compare(st["depths"], f["depth"], vis),
         "means2D": gr.compare(st["means2D"], f["means2D"], vis),
         "conic": gr.compare(st["conic_opacity"][:, :3], f["conic"], vis)}
    if factors:
        e["cov3D"] = gr.compare(st["cov3D"], f["cov3D"], ok & ~f["near"])
    if shs is not None:
        e["rgb"] = gr.compare(st["rgb"], f["rgb"], vis)
    b = gr.geom_backward(sc["means3D"], radii, *camargs, cov_pre if not factors else st["cov3D"],
                         grads["dL_dmeans2D"], grads["dL_dconic"], scales=sc["scales"] if factors else None,
                         rotations=sc["rotations"] if factors else None, scale_modifier=mod, shs=shs, D=D,
                         clamped=st.get("clamped"), dL_dcolors=dcolors_view)
    for k in GEOM_GRADS:
        if k in b:
            e[k] = gr.compare(grads[k], b[k], ok)
            assert float(b[k].v.abs().max()) > 0, k
    if not factors:   # no scale / rotation writes
        assert float(grads["dL_dscales"].abs().max()) == 0.0 and float(grads["dL_drotations"].abs().max()) == 0.0
    return e, float(f["fragile"][~f["near"]].double().mean()), f


def check_views(scene, cams, bg, *, dl_offset=0, feat_offset=0, dcolors_offset=0, tile_rows=None, seed=0,
                sh_degree=None, M=16, cov3D_precomp=None, scale_modifier=1.0, offsets=None, geometry=True,
                blend=True):
    """Forward and backward of len(cams) views of `scene` in one sgb_*_batch call sequence on a fresh ctx, each view
    checked against the float64 restatements on its own state.  Colours are scene.features as colors_precomp, or
    with sh_degree = D the first M coefficients of scene.shs.  cov3D_precomp (P, 6) replaces scales / rotations.
    offsets maps "means3D", "scales", "rotations", "shs", "dL_drotations" to a byte offset off 16-byte alignment.
    dL/dout is random, zero at blend-fragile pixels and, with tile_rows, outside those tile rows; blend=False skips
    the blend restatement (dL/dout random everywhere) and checks the geometry alone.  Returns per-case statistics:
    compare() of every output (<= 1 passes), fragile fractions, list lengths, the weight-pool chunks, the radii and
    (geom) the geometry restatement's forward of the first view."""
    lib = _lib.load()
    W, H = cams[0].image_width, cams[0].image_height
    P = scene.xyz.shape[0]
    use_sh = sh_degree is not None
    Cn = 3 if use_sh else scene.features.shape[1]
    V = len(cams)
    offsets = dict(offsets or {})
    sc = dev_scene(scene, DEV)
    for k in ("means3D", "scales", "rotations"):
        sc[k] = _placed(sc[k], offsets.get(k, 0))
    shs = _placed(sc["shs"][:, :M].contiguous(), offsets.get("shs", 0)) if use_sh else None
    feats = None if use_sh else _placed(sc["features"], feat_offset)
    cov_pre = None if cov3D_precomp is None else torch.as_tensor(cov3D_precomp, dtype=torch.float32, device=DEV)
    bg = torch.as_tensor(bg, dtype=torch.float32, device=DEV)
    cms = [dev_cam(c, DEV) for c in cams]
    ptr = lambda t: None if t is None else t.data_ptr()
    inp = _lib.ViewInputs(
        P=P, D=sh_degree if use_sh else 0, M=M if use_sh else 0, W=W, H=H, C=Cn, background=bg.data_ptr(),
        means3D=sc["means3D"].data_ptr(), shs=ptr(shs), colors_precomp=ptr(feats), opacities=sc["opacities"].data_ptr(),
        scales=None if cov_pre is not None else sc["scales"].data_ptr(), scale_modifier=scale_modifier,
        rotations=None if cov_pre is not None else sc["rotations"].data_ptr(), cov3D_precomp=ptr(cov_pre),
        viewmatrix=None, projmatrix=None, campos=None, tan_fovx=0.0, tan_fovy=0.0, prefiltered=0, debug=0)
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
        img = [torch.empty((lib.sgb_image_bytes(W, H),), **u8) for _ in cams]
        Rs = (Ct.c_int64 * V)()
        _lib.check(lib.sgb_forward_geometry_batch(ctx, Ct.byref(inp), V, cam_arr, ptrs(geom), ptrs(radii), Rs, stream),
                   "sgb_forward_geometry_batch")
        binning = [torch.empty((lib.sgb_binning_bytes(R),), **u8) for R in Rs]
        color = [torch.empty((Cn, H, W), device=DEV) for _ in cams]
        _lib.check(lib.sgb_forward_render_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(geom), ptrs(binning),
                                                ptrs(img), ptrs(radii), ptrs(color), None, stream),
                   "sgb_forward_render_batch")
        chunks = lib.sgb_ctx_view_stat(ctx, 1)

        # the float64 forward of every view on the kernel's own state; dL/dout from it
        g = torch.Generator(device=DEV).manual_seed(seed)
        geo_fields = ("depths", "cov3D", "rgb", "clamped", "tiles_touched") if geometry else ()
        views, dLs = [], []
        for v in range(V):
            R = Rs[v]
            if R == 0:
                views.append(None)
                dLs.append(torch.randn((Cn, H, W), device=DEV, generator=g))
                continue
            st = read_state(lib, P, R, W, H, geom[v], binning[v], img[v], geo_fields + (("rgb",) if use_sh else ()))
            feat_v = st["rgb"] if use_sh else sc["features"]
            args = (st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], feat_v, bg, W, H)
            dL = torch.randn((Cn, H * W), device=DEV, generator=g)
            want = None
            if blend:
                want = br.blend_forward(*args, tile_rows=tile_rows)
                dL[:, want["fragile"]] = 0.0
                if tile_rows is not None:
                    dL[:, :tile_rows[0] * 16 * W] = 0.0
                    dL[:, tile_rows[1] * 16 * W:] = 0.0
            views.append((st, args, want))
            dLs.append(dL.reshape(Cn, H, W))
        dL_in = [_placed(d, dl_offset) for d in dLs]
        z = lambda *s: torch.zeros(s, device=DEV)
        # colors_precomp: one dL_dcolors shared by the views (the gradient a data-parallel step exchanges); SH: one
        # per view, as sgb_backward_batch requires
        shared = _placed(z(P, Cn), dcolors_offset)
        dcolors = [_placed(z(P, Cn), dcolors_offset) for _ in cams] if use_sh else [shared] * V
        grads = [dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 4), dL_dopacity=z(P), dL_dcolors=dcolors[v],
                      dL_dmeans3D=z(P, 3), dL_dcov3D=z(P, 6), dL_dsh=z(P, M, 3) if use_sh else None,
                      dL_dscales=z(P, 3), dL_drotations=_placed(z(P, 4), offsets.get("dL_drotations", 0)))
                 for v in range(V)]
        gr_arr = (_lib.ViewGrads * V)(*[_lib.ViewGrads(**{k: ptr(t) for k, t in gv.items()}) for gv in grads])
        _lib.check(lib.sgb_backward_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(radii), ptrs(geom), ptrs(binning),
                                          ptrs(img), ptrs(dL_in), gr_arr, stream), "sgb_backward_batch")
    finally:
        torch.cuda.synchronize(DEV)
        lib.sgb_ctx_destroy(ctx)

    errs = {}
    frag, gfrag, lens, geo = [], [], [], []
    want_colors = torch.zeros((P, Cn), dtype=torch.float64, device=DEV)
    geo_inp = dict(shs=shs, D=sh_degree if use_sh else 0, scale_modifier=scale_modifier, cov3D_precomp=cov_pre)
    merge = lambda e: errs.update({k: max(errs.get(k, 0.0), x) for k, x in e.items()})
    for v in range(V):
        if views[v] is None:   # nothing in view: the image is the background, no gradient
            assert torch.equal(color[v], bg[:, None, None].expand(Cn, H, W))
            for name in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D"):
                assert float(grads[v][name].abs().max()) == 0.0, name
            continue
        st, args, want = views[v]
        rg = st["ranges"].long()
        lens.append(rg[:, 1] - rg[:, 0])
        if geometry:
            e, gf, fv = _geometry_errors(sc, cams[v], W, H, geo_inp, st, radii[v], grads[v],
                                        dcolors[v] if use_sh else None)
            merge(e)
            gfrag.append(gf)
            geo.append(fv)
        if not blend:
            continue
        wb = br.blend_backward(*args, dLs[v], tile_rows=tile_rows)
        want_colors += wb["dL_dcolors"]
        fragile = want["fragile"]
        ok = ~fragile
        if tile_rows is not None:
            ok[:tile_rows[0] * 16 * W] = False
            ok[tile_rows[1] * 16 * W:] = False
        frag.append(float(fragile[ok | fragile].double().mean()))
        assert torch.equal(st["n_contrib"][ok].long(), want["n_contrib"][ok]), v
        got_grads = {k: grads[v][k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity")}
        got_grads["dL_dcolors"] = wb["dL_dcolors"]   # a shared buffer is checked against the sum below
        e = dict(final_T=br.compare(st["final_T"][ok], want["final_T"][ok]),
                 color=br.compare(color[v].reshape(Cn, -1)[:, ok], want["color"].reshape(Cn, -1)[:, ok]))
        e.update({k: x for k, x in br.grad_errors(got_grads, wb).items() if k != "dL_dcolors"})
        if use_sh:
            e["dL_dcolors"] = br.compare(dcolors[v], wb["dL_dcolors"])
        merge(e)
        for name in ("dL_dmeans2D", "dL_dconic", "dL_dopacity"):
            assert float(wb[name].abs().max()) > 0, name
    if blend and not use_sh:
        errs["dL_dcolors"] = br.compare(shared, want_colors)
        assert float(want_colors.abs().max()) > 0
    first = next((x for x in views if x is not None), None)
    return dict(errs=errs, fragile=max(frag, default=0.0), geom_fragile=max(gfrag, default=0.0),
                lens=torch.cat(lens).cpu() if lens else torch.zeros(0), chunks=chunks, radii=[r.cpu() for r in radii],
                n_contrib=views[0][0]["n_contrib"].cpu() if views[0] else None, W=W, H=H,
                first_state=first[0] if first else None, geom=geo[0] if geo else None)


def report(tag, name, res, t0):
    e = " ".join(f"{k}={v:.3g}" for k, v in res["errs"].items())
    print(f"\n[fp64 {tag}] {name}: fragile={res['fragile']:.4%} geom_fragile={res['geom_fragile']:.4%} {e} "
          f"({time.time() - t0:.1f} s)")


def assert_ok(res):
    assert res["fragile"] <= FRAGILE_MAX, res["fragile"]
    assert res["geom_fragile"] <= FRAGILE_MAX, res["geom_fragile"]
    assert all(v <= 1.0 for v in res["errs"].values()), res["errs"]
