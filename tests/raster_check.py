"""The kernels of one forward + backward against the float64 restatements, through the C ABI: the blend
(tests/blend_ref.py) and the per-Gaussian geometry (tests/geom_ref.py).  Both restatements run on the kernels' own
state (sgb_state_field) and, in the backward, on the kernels' own upstream gradients, so the only error measured is
each stage's own arithmetic.  With anti-aliasing the geometry kernel overwrites dL_dopacity (dL/d(o h), the
blends' sum) with dL/do = h dL/d(o h); the geometry restatement gets the kernel's own dL/d(o h) back as
dL_dopacity / |h| with the h the forward stored ("aa_h").  The joint render (sgb_*_joint_batch) is checked as three
blends over one walk: RGB, the feature table and, with exp_alpha, E / A as the blend of [depth, 1] over 0."""
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
    geometry fields ("depths", "cov3D", "rgb", "clamped", "tiles_touched", "aa_h")."""
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    spec = dict(means2D=(torch.float32, (P, 2)), conic_opacity=(torch.float32, (P, 4)),
                point_list=(torch.int32, (max(R, 1),)), ranges=(torch.int32, (tiles, 2)),
                n_contrib=(torch.int32, (H * W,)), final_T=(torch.float32, (H * W,)))
    extra = dict(depths=(torch.float32, (P,)), cov3D=(torch.float32, (P, 6)), rgb=(torch.float32, (P, 3)),
                 clamped=(torch.uint8, (P, 3)), tiles_touched=(torch.int32, (P,)), aa_h=(torch.float32, (P,)))
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


def _geometry_errors(sc, cam, W, H, inp_args, st, radii, grads, dcolors_view, antialiasing=False, mutation=None):
    """Every forward geometry field and every geometry gradient of one view against geom_ref (its backward with
    `mutation`, one of geom_ref.AA_MUTATIONS, or none).  Returns (errors, fragile fraction, forward restatement).
    With anti-aliasing, dL_dopacity here checks the h the kernel stored against the restatement's (g is recovered
    through it).  That the kernel multiplied the blends' g by that h is checked by check_views' blend comparison
    and, above the floor, by the covariance term the recovered g feeds."""
    shs, D, mod, cov_pre = inp_args["shs"], inp_args["D"], inp_args["scale_modifier"], inp_args["cov3D_precomp"]
    aa = antialiasing
    factors = cov_pre is None
    camargs = (cam.world_view_transform, cam.full_proj_transform, cam.camera_center, W, H,
               math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5))
    f = gr.geom_forward(sc["means3D"], sc["opacities"], *camargs, scales=sc["scales"] if factors else None,
                        rotations=sc["rotations"] if factors else None, scale_modifier=mod, cov3D_precomp=cov_pre,
                        shs=shs, D=D, antialiasing=aa)
    ok = ~f["fragile"]
    vis = f["visible"] & ok
    # integers: equal except on fragile Gaussians
    assert torch.equal(radii.long()[ok], f["radii"][ok])
    assert torch.equal(st["tiles_touched"].long()[ok], f["tiles_touched"][ok])
    if shs is not None:
        assert torch.equal(st["clamped"].bool()[vis], f["clamped"][vis])
    e = {"depth": gr.compare(st["depths"], f["depth"], vis),
         "means2D": gr.compare(st["means2D"], f["means2D"], vis),
         "conic": gr.compare(st["conic_opacity"][:, :3], f["conic"], vis)}
    if aa:   # the record's opacity is o h, its fourth float the signed h (negative on the floor branch)
        hk = st["aa_h"]
        assert torch.equal(hk[vis] > 0, f["aa_active"][vis])
        e["aa_h"] = gr.compare(hk.abs(), f["aa_h"], vis)
        e["aa_opacity"] = gr.compare(st["conic_opacity"][:, 3], f["aa_opacity"], vis)
    else:
        assert torch.equal(st["conic_opacity"][vis, 3], sc["opacities"].reshape(-1)[vis])
    if factors:
        e["cov3D"] = gr.compare(st["cov3D"], f["cov3D"], ok & ~f["near"])
    if shs is not None:
        e["rgb"] = gr.compare(st["rgb"], f["rgb"], vis)
    aa_kw = {}
    if aa:   # the kernel's own dL/d(o h): what the blends wrote, before the geometry kernel scaled it by h
        live = radii > 0
        g_oh = torch.where(live, grads["dL_dopacity"].reshape(-1).double() / st["aa_h"].abs().double().clamp(min=1e-30),
                           torch.zeros_like(grads["dL_dopacity"].reshape(-1).double()))
        aa_kw = dict(antialiasing=True, opacities=sc["opacities"], dL_dopacity=g_oh)
    b = gr.geom_backward(sc["means3D"], radii, *camargs, cov_pre if not factors else st["cov3D"],
                         grads["dL_dmeans2D"], grads["dL_dconic"], scales=sc["scales"] if factors else None,
                         rotations=sc["rotations"] if factors else None, scale_modifier=mod, shs=shs, D=D,
                         clamped=st.get("clamped"), dL_dcolors=dcolors_view, mutation=mutation, **aa_kw)
    if aa:
        e["dL_dopacity"] = gr.compare(grads["dL_dopacity"], b["dL_dopacity"], ok)
    for k in GEOM_GRADS:
        if k in b:
            e[k] = gr.compare(grads[k], b[k], ok)
            assert float(b[k].v.abs().max()) > 0, k
    if not factors:   # no scale / rotation writes
        assert float(grads["dL_dscales"].abs().max()) == 0.0 and float(grads["dL_drotations"].abs().max()) == 0.0
    return e, float(f["fragile"][~f["near"]].double().mean()), f


def _joint_errors(st, args, ok, features, bg_features, fimg, dF, ea, tile_rows):
    """The joint render's extra images of one view over the walk of `args` (blend_forward's arguments for RGB): the
    feature image of (features, bg_features) and, with ea = (E, A, dL/d(E, A)), E / A as the blend of [depth, 1] over
    0.  Returns (errors at the pixels ok, [feature blend backward, (E / A blend backward)])."""
    fargs = args[:4] + (features, bg_features) + args[6:]
    fw = br.blend_forward(*fargs, tile_rows=tile_rows)
    c = features.shape[1]
    e = {"features": br.compare(fimg.reshape(c, -1)[:, ok], fw["color"].reshape(c, -1)[:, ok])}
    parts = [br.blend_backward(*fargs, dF, tile_rows=tile_rows)]
    if ea is not None:
        E, A, dEA = ea
        za = torch.stack([st["depths"], torch.ones_like(st["depths"])], 1)
        eargs = args[:4] + (za, torch.zeros(2, dtype=torch.float32, device=DEV)) + args[6:]
        ew = br.blend_forward(*eargs, tile_rows=tile_rows)
        e["exp_alpha"] = br.compare(torch.cat([E, A]).reshape(2, -1)[:, ok], ew["color"].reshape(2, -1)[:, ok])
        parts.append(br.blend_backward(*eargs, dEA, tile_rows=tile_rows))
    return e, parts


# kernel bugs of the anti-aliased opacity gradient, applied to the kernel's output (check_views' mutation): a
# geometry kernel that writes the blends' g, or h^2 g, into dL_dopacity instead of h g
KERNEL_MUTATIONS = ("kernel_dopacity_unscaled", "kernel_dopacity_h_squared")


def check_views(scene, cams, bg, *, dl_offset=0, feat_offset=0, dcolors_offset=0, tile_rows=None, seed=0,
                sh_degree=None, M=16, cov3D_precomp=None, scale_modifier=1.0, offsets=None, geometry=True,
                blend=True, antialiasing=False, joint=None, exp_alpha=False, fresh_backward_ctx=False, mutation=None):
    """Forward and backward of len(cams) views of `scene` in one sgb_*_batch call sequence on a fresh ctx, each view
    checked against the float64 restatements on its own state.  Colours are scene.features as colors_precomp, or
    with sh_degree = D the first M coefficients of scene.shs.  cov3D_precomp (P, 6) replaces scales / rotations.
    offsets maps "means3D", "scales", "rotations", "shs", "dL_drotations" to a byte offset off 16-byte alignment.
    dL/dout is random, zero at blend-fragile pixels and, with tile_rows, outside those tile rows; blend=False skips
    the blend restatement (dL/dout random everywhere) and checks the geometry alone.  antialiasing sets
    sgb_view_inputs.antialiasing.  joint = (features (P, c), bg_features (c,)) renders and differentiates them with
    the RGB image through sgb_*_joint_batch (the RGB colours as above, C = 3; feat_offset then places the feature
    table and dcolors_offset dL_dfeatures too); exp_alpha adds E / A and their upstream gradients (the geometry
    restatement is then skipped: their dL/dz stays in ctx scratch); fresh_backward_ctx runs the backward on a second
    ctx, which must rebuild the weight pool.  mutation, to show that the comparison rejects a bug: one of
    geom_ref.AA_MUTATIONS (the restatement's backward mutated) or of KERNEL_MUTATIONS (the kernel's dL_dopacity
    rewritten as a kernel with that bug would have written it).  Returns per-case statistics: compare() of every
    output (<= 1 passes), fragile fractions, list lengths, the weight-pool chunks, the radii and (geom) the geometry
    restatement's forward of the first view."""
    lib = _lib.load()
    W, H = cams[0].image_width, cams[0].image_height
    P = scene.xyz.shape[0]
    use_sh = sh_degree is not None
    Cn = 3 if use_sh else scene.features.shape[1]
    V = len(cams)
    offsets = dict(offsets or {})
    assert joint is not None or not (exp_alpha or fresh_backward_ctx)
    assert mutation is None or (antialiasing and mutation in gr.AA_MUTATIONS + KERNEL_MUTATIONS), mutation
    sc = dev_scene(scene, DEV)
    for k in ("means3D", "scales", "rotations"):
        sc[k] = _placed(sc[k], offsets.get(k, 0))
    shs = _placed(sc["shs"][:, :M].contiguous(), offsets.get("shs", 0)) if use_sh else None
    feats = None if use_sh else _placed(sc["features"], 0 if joint is not None else feat_offset)
    if joint is not None:
        assert Cn == 3
        jf = _placed(torch.as_tensor(joint[0], dtype=torch.float32, device=DEV).contiguous(), feat_offset)
        jbg = torch.as_tensor(joint[1], dtype=torch.float32, device=DEV).contiguous()
        c = jf.shape[1]
    cov_pre = None if cov3D_precomp is None else torch.as_tensor(cov3D_precomp, dtype=torch.float32, device=DEV)
    bg = torch.as_tensor(bg, dtype=torch.float32, device=DEV)
    cms = [dev_cam(c_, DEV) for c_ in cams]
    ptr = lambda t: None if t is None else t.data_ptr()
    inp = _lib.ViewInputs(
        P=P, D=sh_degree if use_sh else 0, M=M if use_sh else 0, W=W, H=H, C=Cn, background=bg.data_ptr(),
        means3D=sc["means3D"].data_ptr(), shs=ptr(shs), colors_precomp=ptr(feats), opacities=sc["opacities"].data_ptr(),
        scales=None if cov_pre is not None else sc["scales"].data_ptr(), scale_modifier=scale_modifier,
        rotations=None if cov_pre is not None else sc["rotations"].data_ptr(), cov3D_precomp=ptr(cov_pre),
        viewmatrix=None, projmatrix=None, campos=None, tan_fovx=0.0, tan_fovy=0.0, prefiltered=0, debug=0,
        antialiasing=int(bool(antialiasing)))
    cam_arr = (_lib.Camera * V)(*[_lib.Camera(c_["viewmatrix"].data_ptr(), c_["projmatrix"].data_ptr(),
                                              c_["campos"].data_ptr(), c_["tanfovx"], c_["tanfovy"]) for c_ in cms])
    ptrs = lambda ts: (Ct.c_void_p * V)(*[t.data_ptr() for t in ts])
    u8 = dict(dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    ctx, ctx_b = Ct.c_void_p(), Ct.c_void_p()
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
        if joint is None:
            _lib.check(lib.sgb_forward_render_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(geom), ptrs(binning),
                                                    ptrs(img), ptrs(radii), ptrs(color), None, stream),
                       "sgb_forward_render_batch")
        else:
            depth = [torch.empty((1, H, W), device=DEV) for _ in cams]
            ea = [[torch.empty((1, H, W), device=DEV) for _ in cams] for _ in range(2)] if exp_alpha else None
            fimg = [torch.empty((c, H, W), device=DEV) for _ in cams]
            _lib.check(lib.sgb_forward_render_joint_batch(
                ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(geom), ptrs(binning), ptrs(img), ptrs(radii), ptrs(color),
                ptrs(depth), ptrs(ea[0]) if exp_alpha else None, ptrs(ea[1]) if exp_alpha else None, jf.data_ptr(), c,
                jbg.data_ptr(), ptrs(fimg), stream), "sgb_forward_render_joint_batch")
        chunks = lib.sgb_ctx_view_stat(ctx, 1)

        # the float64 forward of every view on the kernel's own state; dL/dout from it
        g = torch.Generator(device=DEV).manual_seed(seed)
        geo_fields = ("depths", "cov3D", "rgb", "clamped", "tiles_touched", "aa_h") if geometry else ()
        if exp_alpha:
            geo_fields += ("depths",)
        views, dLs, dFs, dEAs = [], [], [], []
        for v in range(V):
            R = Rs[v]
            if R == 0:
                views.append(None)
                dLs.append(torch.randn((Cn, H, W), device=DEV, generator=g))
                if joint is not None:
                    dFs.append(torch.randn((c, H, W), device=DEV, generator=g))
                    dEAs.append(torch.randn((2, H, W), device=DEV, generator=g))
                continue
            st = read_state(lib, P, R, W, H, geom[v], binning[v], img[v],
                            tuple(dict.fromkeys(geo_fields + (("rgb",) if use_sh else ()))))
            feat_v = st["rgb"] if use_sh else sc["features"]
            args = (st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], feat_v, bg, W, H)
            dL = torch.randn((Cn, H * W), device=DEV, generator=g)
            extra = []
            if joint is not None:
                extra = [torch.randn((n, H * W), device=DEV, generator=g) for n in (c, 2)]
            want = None
            if blend:
                want = br.blend_forward(*args, tile_rows=tile_rows)
                for d in [dL] + extra:   # the walk's fragile pixels are the same for every table blended over it
                    d[:, want["fragile"]] = 0.0
                    if tile_rows is not None:
                        d[:, :tile_rows[0] * 16 * W] = 0.0
                        d[:, tile_rows[1] * 16 * W:] = 0.0
            views.append((st, args, want))
            dLs.append(dL.reshape(Cn, H, W))
            if joint is not None:
                dFs.append(extra[0].reshape(c, H, W))
                dEAs.append(extra[1].reshape(2, H, W))
        dL_in = [_placed(d, dl_offset) for d in dLs]
        z = lambda *s_: torch.zeros(s_, device=DEV)
        # colors_precomp: one dL_dcolors shared by the views (the gradient a data-parallel step exchanges); SH: one
        # per view, as sgb_backward_batch requires
        shared = _placed(z(P, Cn), dcolors_offset)
        dcolors = [_placed(z(P, Cn), dcolors_offset) for _ in cams] if use_sh else [shared] * V
        grads = [dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 4), dL_dopacity=z(P), dL_dcolors=dcolors[v],
                      dL_dmeans3D=z(P, 3), dL_dcov3D=z(P, 6), dL_dsh=z(P, M, 3) if use_sh else None,
                      dL_dscales=z(P, 3), dL_drotations=_placed(z(P, 4), offsets.get("dL_drotations", 0)))
                 for v in range(V)]
        gr_arr = (_lib.ViewGrads * V)(*[_lib.ViewGrads(**{k: ptr(t) for k, t in gv.items()}) for gv in grads])
        bctx = ctx
        if fresh_backward_ctx:   # the forward's weight pool is not there: the backward rebuilds it
            _lib.check(lib.sgb_ctx_create(Ct.byref(ctx_b), DEV.index), "sgb_ctx_create")
            bctx = ctx_b
        if joint is None:
            _lib.check(lib.sgb_backward_batch(bctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(radii), ptrs(geom),
                                              ptrs(binning), ptrs(img), ptrs(dL_in), gr_arr, stream),
                       "sgb_backward_batch")
        else:
            dE = [d[0:1].contiguous() for d in dEAs] if exp_alpha else None
            dA = [d[1:2].contiguous() for d in dEAs] if exp_alpha else None
            dfeat_in = [d.contiguous() for d in dFs]
            dL_dfeatures = _placed(z(P, c), dcolors_offset)
            _lib.check(lib.sgb_backward_joint_batch(
                bctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(radii), ptrs(geom), ptrs(binning), ptrs(img), ptrs(dL_in),
                ptrs(dE) if exp_alpha else None, ptrs(dA) if exp_alpha else None, gr_arr, jf.data_ptr(), c,
                jbg.data_ptr(), ptrs(dfeat_in), dL_dfeatures.data_ptr(), stream), "sgb_backward_joint_batch")
    finally:
        torch.cuda.synchronize(DEV)
        lib.sgb_ctx_destroy(ctx)
        if ctx_b.value:
            lib.sgb_ctx_destroy(ctx_b)

    errs = {}
    frag, gfrag, lens, geo = [], [], [], []
    want_colors = torch.zeros((P, Cn), dtype=torch.float64, device=DEV)
    want_dfeat = torch.zeros((P, c), dtype=torch.float64, device=DEV) if joint is not None else None
    geo_inp = dict(shs=shs, D=sh_degree if use_sh else 0, scale_modifier=scale_modifier, cov3D_precomp=cov_pre)
    merge = lambda e: errs.update({k: max(errs.get(k, 0.0), x) for k, x in e.items()})
    if mutation in KERNEL_MUTATIONS:
        for v in range(V):
            if views[v] is not None:
                h_k = torch.where(radii[v] > 0, views[v][0]["aa_h"].abs(), torch.ones_like(grads[v]["dL_dopacity"]))
                d = grads[v]["dL_dopacity"]
                d.copy_(d / h_k if mutation == "kernel_dopacity_unscaled" else d * h_k)
    for v in range(V):
        if views[v] is None:   # nothing in view: the image is the background, no gradient
            assert torch.equal(color[v], bg[:, None, None].expand(Cn, H, W))
            if joint is not None:
                assert torch.equal(fimg[v], jbg[:, None, None].expand(c, H, W))
                if exp_alpha:
                    assert not ea[0][v].any() and not ea[1][v].any()
            for name in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D"):
                assert float(grads[v][name].abs().max()) == 0.0, name
            continue
        st, args, want = views[v]
        rg = st["ranges"].long()
        lens.append(rg[:, 1] - rg[:, 0])
        if geometry and not exp_alpha:
            e, gf, fv = _geometry_errors(sc, cams[v], W, H, geo_inp, st, radii[v], grads[v],
                                        dcolors[v] if use_sh else None, antialiasing,
                                        mutation if mutation in gr.AA_MUTATIONS else None)
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
        e = dict(final_T=br.compare(st["final_T"][ok], want["final_T"][ok]),
                 color=br.compare(color[v].reshape(Cn, -1)[:, ok], want["color"].reshape(Cn, -1)[:, ok]))
        # the blend gradients of every image blended over this walk, summed as the kernels sum them
        want_g = {k: wb[k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity")}
        if joint is not None:
            je, parts = _joint_errors(st, args, ok, jf, jbg, fimg[v], dFs[v],
                                      (ea[0][v], ea[1][v], dEAs[v]) if exp_alpha else None, tile_rows)
            e.update(je)
            want_dfeat += parts[0]["dL_dcolors"]
            for part in parts:
                for k in want_g:
                    want_g[k] = want_g[k] + part[k]
        if antialiasing:   # the geometry kernel scaled the blends' dL/d(o h) by the h the forward stored
            h_k = torch.where(radii[v] > 0, st["aa_h"].abs().double(), torch.zeros_like(want_g["dL_dopacity"]))
            want_g["dL_dopacity"] = want_g["dL_dopacity"] * h_k
        got_grads = {k: grads[v][k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity")}
        got_grads["dL_dcolors"] = wb["dL_dcolors"]   # a shared buffer is checked against the sum below
        want_g["dL_dcolors"] = wb["dL_dcolors"]
        e.update({k: x for k, x in br.grad_errors(got_grads, want_g).items() if k != "dL_dcolors"})
        if use_sh:
            e["dL_dcolors"] = br.compare(dcolors[v], wb["dL_dcolors"])
        merge(e)
        for name in ("dL_dmeans2D", "dL_dconic", "dL_dopacity"):
            assert float(want_g[name].abs().max()) > 0, name
    if blend and not use_sh:
        errs["dL_dcolors"] = br.compare(shared, want_colors)
        assert float(want_colors.abs().max()) > 0
    if blend and joint is not None:
        errs["dL_dfeatures"] = br.compare(dL_dfeatures, want_dfeat)
        assert float(want_dfeat.abs().max()) > 0
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
