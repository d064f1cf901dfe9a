"""Autograd boundary of the rasterizer: the Python surface of the reference's two extensions
(``channel_rasterization/__init__.py`` and ``rgbd_rasterization/__init__.py``) over libsgb200.

``_C_chn`` / ``_C_rgbd`` reproduce the pybind entry points ``rasterize_gaussians``,
``rasterize_gaussians_backward`` and ``mark_visible`` (ext.cpp:16-18) with the reference's
positional argument lists and return tuples; ``make_module`` builds the
GaussianRasterizationSettings / GaussianRasterizer / _RasterizeGaussians trio for each variant.
A single view is the V = 1 case of the batched native calls, as in the C library (api.cu).
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# The batched entry points take one entry per view behind a pointer.  ctypes passes a single instance by reference,
# which spares the common one-view call from building arrays.
def _ptrs(ts):
    if len(ts) == 1:
        return C.c_void_p(ts[0].data_ptr())
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _per_view(ctype, items):
    return items[0] if len(items) == 1 else (ctype * len(items))(*items)


def _opt(t: Optional[torch.Tensor], device, what: str) -> Optional[torch.Tensor]:
    """The reference encodes an absent optional input as an empty tensor → nullptr
    (channel_rasterization/__init__.py:266-276, rasterize_points.cu:99-117)."""
    if t is None or t.numel() == 0:
        return None
    return _f32(t, device, what)


def _f32(t: torch.Tensor, device, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor")
    if t.device != device:
        raise ValueError(f"{what} is on {t.device}, expected {device}")
    if t.dtype != torch.float32:
        raise TypeError(f"{what} must be float32, got {t.dtype}")
    return t.contiguous()


def _stream_ctx(device):
    s = torch.cuda.current_stream(device).cuda_stream
    return s, _lib.ctx_for(device.index if device.index is not None else torch.cuda.current_device(), s)


def _make_inputs(cams, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                 H, W, sh, degree, prefiltered, debug, num_channels, antialiasing=False):
    """``cams`` holds one (viewmatrix, projmatrix, campos, tan_fovx, tan_fovy) per view.  Returns the shared inputs
    (carrying view 0's camera), the sgb_camera array, the tensors both point into, and the device.  ``antialiasing``:
    the opacity-compensated screen-space filter (sgb_view_inputs.antialiasing)."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:61-64
    if not means3D.is_cuda:
        raise RuntimeError("means3D must be a CUDA tensor: the rasterizer has no CPU path")
    dev = means3D.device
    viewmatrix, projmatrix, campos, tan_fovx, tan_fovy = cams[0]
    keep = dict(
        background=_f32(background, dev, "bg"), means3D=_f32(means3D, dev, "means3D"),
        colors=_opt(colors, dev, "colors_precomp"), opacity=_f32(opacity, dev, "opacities"),
        scales=_opt(scales, dev, "scales"), rotations=_opt(rotations, dev, "rotations"),
        cov3D=_opt(cov3D_precomp, dev, "cov3D_precomp"), view=_f32(viewmatrix, dev, "viewmatrix"),
        proj=_f32(projmatrix, dev, "projmatrix"), sh=_opt(sh, dev, "shs"), campos=_f32(campos, dev, "campos"))
    P = means3D.size(0)
    M = keep["sh"].size(1) if keep["sh"] is not None else 0  # rasterize_points.cu:88-92
    if keep["background"].numel() < num_channels:
        raise RuntimeError(f"bg has {keep['background'].numel()} entries, need {num_channels}")
    if keep["colors"] is not None and keep["colors"].shape != (P, num_channels):
        raise RuntimeError(f"colors_precomp must be ({P}, {num_channels}), got {tuple(keep['colors'].shape)}")
    inp = _lib.ViewInputs(
        P=P, D=int(degree), M=int(M), W=int(W), H=int(H), C=int(num_channels),
        background=_ptr(keep["background"]), means3D=_ptr(keep["means3D"]), shs=_ptr(keep["sh"]),
        colors_precomp=_ptr(keep["colors"]), opacities=_ptr(keep["opacity"]), scales=_ptr(keep["scales"]),
        scale_modifier=float(scale_modifier), rotations=_ptr(keep["rotations"]),
        cov3D_precomp=_ptr(keep["cov3D"]), viewmatrix=_ptr(keep["view"]), projmatrix=_ptr(keep["proj"]),
        campos=_ptr(keep["campos"]), tan_fovx=float(tan_fovx), tan_fovy=float(tan_fovy),
        prefiltered=int(bool(prefiltered)), debug=int(bool(debug)), antialiasing=int(bool(antialiasing)))
    # view 0 is the camera of the shared inputs, checked above in the reference's argument order
    cameras = [_lib.Camera(inp.viewmatrix, inp.projmatrix, inp.campos, inp.tan_fovx, inp.tan_fovy)]
    for v, (viewmatrix, projmatrix, campos, tan_fovx, tan_fovy) in enumerate(cams[1:], 1):
        keep[v] = (_f32(viewmatrix, dev, "viewmatrix"), _f32(projmatrix, dev, "projmatrix"),
                   _f32(campos, dev, "campos"))
        cameras.append(_lib.Camera(*[t.data_ptr() for t in keep[v]], float(tan_fovx), float(tan_fovy)))
    return inp, _per_view(_lib.Camera, cameras), keep, dev


def _forward(want_depth: bool, what: str, cams, background, means3D, colors, opacity, scales, rotations,
             scale_modifier, cov3D_precomp, image_height, image_width, sh, degree, prefiltered, debug, num_channels,
             want_exp_alpha=False, features=None, bg_features=None, antialiasing=False):
    """V = len(cams) views of the same Gaussians through sgb_forward_geometry_batch / sgb_forward_render_batch_ext:
    one stream sync for all instance counts, one for all weight-pool checks.  With ``features`` (P, c) over
    ``bg_features`` (c), the render call is sgb_forward_render_joint_batch, which also renders that table from the same
    geometry and binning (the RGB render: ``want_depth`` and num_channels = 3).  Returns the marshalled inputs (None
    for an empty scene), which _backward takes, and the per-view lists (R, color, radii, geometry state, binning
    state, image state, depth or None, expected depth or None, alpha or None), followed with ``features`` by the
    per-view list of feature images."""
    lib = _lib.load()
    V = len(cams)
    if features is not None and (features.ndim != 2 or features.size(0) != means3D.size(0) or features.size(1) < 1):
        raise ValueError(f"features must be (P, c) with P = {means3D.size(0)} and c >= 1, got {tuple(features.shape)}")
    if means3D.ndimension() == 2 and means3D.size(0) == 0 and means3D.is_cuda:
        # Empty scene: the reference never enters the native forward (rasterize_points.cu:84) and
        # returns its zero-initialised outputs — zeros, not the background.
        dev = means3D.device
        z = lambda *shape, dtype=torch.float32: [torch.zeros(shape, dtype=dtype, device=dev) for _ in range(V)]
        feat = () if features is None else (z(features.size(1), image_height, image_width),)
        return None, ([0] * V, z(num_channels, image_height, image_width), z(0, dtype=torch.int32),
                      z(0, dtype=torch.uint8), z(0, dtype=torch.uint8),
                      z(lib.sgb_image_bytes(image_width, image_height), dtype=torch.uint8),
                      z(1, image_height, image_width) if want_depth else None,
                      z(1, image_height, image_width) if want_exp_alpha else None,
                      z(1, image_height, image_width) if want_exp_alpha else None, *feat)
    native = _make_inputs(cams, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                          image_height, image_width, sh, degree, prefiltered, debug, num_channels, antialiasing)
    inp, cameras, keep, dev = native
    P, H, W, Cn = inp.P, inp.H, inp.W, inp.C
    if features is not None:
        c = features.size(1)
        feats = _f32(features, dev, "features")
        bg_feats = _f32(bg_features, dev, "bg_features").reshape(-1)
        if bg_feats.numel() != c:
            raise ValueError(f"bg_features has {bg_feats.numel()} entries, the feature table {c} channels")
        keep["features"], keep["bg_features"] = feats, bg_feats
    u8 = dict(dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        stream, ctx = _stream_ctx(dev)
        # every pixel / every radius is written by the kernels: no zero fill (the reference's
        # torch::full of out_color is pure waste, rasterize_points.cu:73)
        out_color = [torch.empty((Cn, H, W), dtype=torch.float32, device=dev) for _ in range(V)]
        out_feat = None if features is None else [torch.empty((c, H, W), dtype=torch.float32, device=dev)
                                                  for _ in range(V)]
        plane = lambda want: [torch.empty((1, H, W), dtype=torch.float32, device=dev) for _ in range(V)] if want else None
        out_depth, out_exp_depth, out_alpha = plane(want_depth), plane(want_exp_alpha), plane(want_exp_alpha)
        radii = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(V)]
        geom = [torch.empty((lib.sgb_geometry_bytes(P),), **u8) for _ in range(V)]
        img = [torch.empty((lib.sgb_image_bytes(W, H),), **u8) for _ in range(V)]
        R = (C.c_int64 * V)()
        # the geometry call waits for the instance counts: only the binning states are left for after it
        geom_p, radii_p, img_p, color_p = _ptrs(geom), _ptrs(radii), _ptrs(img), _ptrs(out_color)
        depth_p = _ptrs(out_depth) if want_depth else None
        exp_p, alpha_p = (_ptrs(out_exp_depth), _ptrs(out_alpha)) if want_exp_alpha else (None, None)
        _lib.check(lib.sgb_forward_geometry_batch(ctx, C.byref(inp), V, cameras, geom_p, radii_p, R, stream),
                   f"{what} (geometry)")
        binning = [torch.empty((lib.sgb_binning_bytes(R[v]),), **u8) for v in range(V)]
        common = (ctx, C.byref(inp), V, cameras, R, geom_p, _ptrs(binning), img_p, radii_p, color_p, depth_p, exp_p,
                  alpha_p)
        if features is None:
            rc = lib.sgb_forward_render_batch_ext(*common, stream)
        else:
            rc = lib.sgb_forward_render_joint_batch(*common, feats.data_ptr(), c, bg_feats.data_ptr(), _ptrs(out_feat),
                                                    stream)
        _lib.check(rc, f"{what} (render)")
    feat = () if features is None else (out_feat,)
    return native, (list(R), out_color, radii, geom, binning, img, out_depth, out_exp_depth, out_alpha, *feat)


def _forward_joint(what: str, cams, background, means3D, colors, opacity, scales, rotations, scale_modifier,
                   cov3D_precomp, image_height, image_width, sh, degree, prefiltered, debug, features, bg_features,
                   want_exp_alpha=False, antialiasing=False):
    """_forward of the RGB render (median depth always) with ``features``: (native, per-view lists as _forward's
    without features, per-view feature images, the marshalled (features, bg_features) or None for an empty scene)."""
    native, (*lists, feat) = _forward(True, what, cams, background, means3D, colors, opacity, scales, rotations,
                                      scale_modifier, cov3D_precomp, image_height, image_width, sh, degree,
                                      prefiltered, debug, 3, want_exp_alpha, features, bg_features, antialiasing)
    return native, tuple(lists), feat, None if native is None else (native[2]["features"], native[2]["bg_features"])


def _backward(what: str, native, radii, dL_dout, geom, R, binning, img, dL_dexp_depth=None, dL_dalpha=None,
              joint=None, cam_grad=False):
    """sgb_backward_batch_ext over the views of one forward: ``native`` is what _make_inputs returned for it, the other
    arguments are per-view lists of its states and of dL/dout (dL/d expected depth and dL/d alpha: per-view lists of
    (1, H, W) planes, or None when absent).  Returns (the per-view list of dL_dmeans2D, then the
    colour, opacity, means3D, cov3D, SH, scale and rotation gradients summed over the views).  Precomputed colours /
    features accumulate over the views in ONE (P, C) buffer inside the kernels; on the SH path the per-view RGB
    gradient is an input of that view's SH backward (backward.cu:385-386), so every view gets its own (P, 3).
    ``joint`` = (features, bg_features, per-view dL/d feature image) runs sgb_backward_joint_batch instead (the forward
    was _forward with ``features``) and appends the (P, c) feature gradient to the result.  ``cam_grad`` runs the
    ``_cam`` entry point of the same call and appends the (V, 35) camera gradients: per view dL/dviewmatrix (16),
    dL/dprojmatrix (16) and dL/dcampos (3) in the element order of the marshalled (contiguous) camera tensors."""
    lib = _lib.load()
    inp, cameras, _, dev = native
    V, P, M, Cn = len(dL_dout), inp.P, inp.M, inp.C
    z = dict(dtype=torch.float32, device=dev)
    shared = M == 0
    # one view has no view axis: its buffers are the gradients, with nothing to index or sum afterwards
    lead = () if V == 1 else (V,)
    g_colors = torch.zeros((P, Cn) if shared else lead + (P, Cn), **z)
    g_means2D, g_conic, g_opacity, g_means3D, g_cov3D, g_sh, g_scales, g_rot = [
        torch.zeros(lead + s, **z) for s in ((P, 3), (P, 2, 2), (P, 1), (P, 3), (P, 6), (P, M, 3), (P, 3), (P, 4))]
    bufs = [g_means2D, g_conic, g_opacity, g_colors, g_means3D, g_cov3D, g_sh, g_scales, g_rot]  # sgb_view_grads order
    gouts = [_f32(g, dev, "dL_dout_color") for g in dL_dout]
    planes = lambda gs, name: None if gs is None else [_f32(g, dev, name).reshape(inp.H, inp.W) for g in gs]
    g_exp, g_alpha = planes(dL_dexp_depth, "dL_dexp_depth"), planes(dL_dalpha, "dL_dalpha")
    g_cam = torch.zeros((V, 35), **z) if cam_grad else None   # an empty scene has a zero camera gradient
    if P != 0:
        # view v's slice of every buffer, by address; the shared colour buffer is the same for all views
        base = [t.data_ptr() for t in bufs]
        if M == 0:
            base[6] = 0  # no SH: dL_dsh stays null
        step = [0 if t is g_colors and shared else t.nbytes // V for t in bufs]
        grads = _per_view(_lib.ViewGrads, [_lib.ViewGrads(*[b + v * s for b, s in zip(base, step)]) for v in range(V)])
        with torch.cuda.device(dev):
            stream, ctx = _stream_ctx(dev)
            num_rendered = (C.c_int64 * V)(*map(int, R))
            common = (ctx, C.byref(inp), V, cameras, num_rendered, _ptrs(radii), _ptrs(geom), _ptrs(binning),
                      _ptrs(img), _ptrs(gouts), None if g_exp is None else _ptrs(g_exp),
                      None if g_alpha is None else _ptrs(g_alpha), grads)
            cams = ()
            if cam_grad:
                b = g_cam.data_ptr()
                cams = (_per_view(_lib.CameraGrads, [_lib.CameraGrads(b + 140 * v, b + 140 * v + 64, b + 140 * v + 128)
                                                     for v in range(V)]),)
            if joint is None:
                fn = lib.sgb_backward_batch_cam if cam_grad else lib.sgb_backward_batch_ext
                _lib.check(fn(*common, *cams, stream), what)
            else:
                feats, bg_feats, gfeat = joint
                g_features = torch.zeros(feats.shape, **z)
                gfeat = [_f32(g, dev, "dL_dfeatures_image") for g in gfeat]
                fn = lib.sgb_backward_joint_batch_cam if cam_grad else lib.sgb_backward_joint_batch
                _lib.check(fn(*common, feats.data_ptr(), feats.size(1), bg_feats.data_ptr(), _ptrs(gfeat),
                              g_features.data_ptr(), *cams, stream), what)
    elif joint is not None:
        g_features = torch.zeros(joint[0].shape, **z)
    summed = [g_colors, g_opacity, g_means3D, g_cov3D, g_sh, g_scales, g_rot]
    tail = (() if joint is None else (g_features,)) + (() if g_cam is None else (g_cam,))
    if V == 1:
        return ([g_means2D], *summed, *tail)
    # the shared colour buffer already holds the sum over the views
    return (list(g_means2D.unbind(0)), *[t if t is g_colors and shared else t.sum(0) for t in summed], *tail)


def _mark_visible(means3D, viewmatrix, projmatrix):
    lib = _lib.load()
    dev = means3D.device
    P = means3D.size(0)
    present = torch.zeros((P,), dtype=torch.bool, device=dev)
    if P != 0:
        m, v, p = _f32(means3D, dev, "positions"), _f32(viewmatrix, dev, "viewmatrix"), _f32(projmatrix, dev, "projmatrix")
        with torch.cuda.device(dev):
            stream, _ = _stream_ctx(dev)
            _lib.check(lib.sgb_mark_visible(P, m.data_ptr(), v.data_ptr(), p.data_ptr(), present.data_ptr(), stream),
                       "mark_visible")
    return present


def _one_view(forward_result):
    """The reference's return tuple from the per-view lists of a single-view _forward."""
    return tuple(x[0] for x in forward_result[1] if x is not None)


class _C_chn:
    """pybind surface of channel_rasterization._C (rasterize_points.cu:38-223, ext.cpp:16-18)."""

    @staticmethod
    def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                            viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree,
                            campos, prefiltered, debug, num_channels):
        return _one_view(_forward(False, "rasterize_gaussians", [(viewmatrix, projmatrix, campos, tan_fovx, tan_fovy)],
                                  background, means3D, colors, opacity, scales, rotations, scale_modifier,
                                  cov3D_precomp, image_height, image_width, sh, degree, prefiltered, debug,
                                  num_channels))

    @staticmethod
    def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh,
                                     degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug):
        Cn, H, W = dL_dout_color.shape  # rasterize_points.cu:146-148
        # opacities are not an input of Rasterizer::backward (they live in the geometry state); the
        # struct field only has to be non-null for validation.
        native = _make_inputs([(viewmatrix, projmatrix, campos, tan_fovx, tan_fovy)], background, means3D, colors,
                              means3D, scales, rotations, scale_modifier, cov3D_precomp, H, W, sh, degree, False, debug,
                              Cn)
        g_means2D, *grads = _backward("rasterize_gaussians_backward", native, [radii], [dL_dout_color], [geomBuffer],
                                      [R], [binningBuffer], [imageBuffer])
        return (g_means2D[0], *grads)

    mark_visible = staticmethod(_mark_visible)


class _C_rgbd:
    """pybind surface of rgbd_rasterization._C (18 / 20 arguments, forward also returns depth)."""

    @staticmethod
    def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                            viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree,
                            campos, prefiltered):
        return _one_view(_forward(True, "rasterize_gaussians", [(viewmatrix, projmatrix, campos, tan_fovx, tan_fovy)],
                                  background, means3D, colors, opacity, scales, rotations, scale_modifier,
                                  cov3D_precomp, image_height, image_width, sh, degree, prefiltered, False, 3))

    @staticmethod
    def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh,
                                     degree, campos, geomBuffer, R, binningBuffer, imageBuffer):
        return _C_chn.rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations,
                                                   scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
                                                   tan_fovy, dL_dout_color, sh, degree, campos, geomBuffer, R,
                                                   binningBuffer, imageBuffer, False)

    mark_visible = staticmethod(_mark_visible)


def _cameras(settings_list):
    return [(rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy) for rs in settings_list]


def _check_batch_settings(settings_list):
    rs0 = settings_list[0]
    if not (1 <= len(settings_list) <= _lib.MAX_BATCH):
        raise ValueError(f"a batch holds 1..{_lib.MAX_BATCH} views, got {len(settings_list)}")
    for rs in settings_list[1:]:
        same = (rs.image_height == rs0.image_height and rs.image_width == rs0.image_width and
                rs.scale_modifier == rs0.scale_modifier and rs.sh_degree == rs0.sh_degree and
                bool(rs.prefiltered) == bool(rs0.prefiltered) and rs.bg is rs0.bg and
                getattr(rs, "num_channels", 3) == getattr(rs0, "num_channels", 3))
        if not same:
            raise ValueError("the views of a batch must share image size, background tensor, scale modifier, SH degree "
                             "and channel count (only the cameras differ)")


def _optional_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp):
    """The reference's argument checks (channel_rasterization/__init__.py:258-276); absent inputs become empty
    tensors."""
    if (shs is None) == (colors_precomp is None):
        raise Exception("Please provide excatly one of either SHs or precomputed colors!")
    if ((scales is None or rotations is None) and cov3D_precomp is None) or (
            (scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    empty = torch.Tensor([])
    return [empty if t is None else t for t in (shs, colors_precomp, scales, rotations, cov3D_precomp)]


def _dump(args, path):
    """Reference debug behaviour without its unconditional CPU deep copy: the argument snapshot is
    taken only when the native call has already failed (channel_rasterization/__init__.py:86-100)."""
    try:
        torch.save(tuple(a.detach().cpu() if isinstance(a, torch.Tensor) else a for a in args), path)
    except Exception:  # pragma: no cover - best effort
        pass


def _native_args(is_chn, joint, settings_list, means3D, sh, colors_precomp, opacities, scales, rotations,
                 cov3Ds_precomp):
    """The _make_inputs arguments of the views in ``settings_list`` (settings of the chn variant when ``is_chn``, of
    the rgbd variant otherwise; ``joint``: of a render that also draws a feature table)."""
    rs = settings_list[0]
    # the rgbd extension's _C takes no debug flag (rgbd_rasterization/__init__.py:57-80); the joint render honours it
    return (_cameras(settings_list), rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
            cov3Ds_precomp, rs.image_height, rs.image_width, sh, rs.sh_degree, rs.prefiltered,
            (is_chn or joint) and rs.debug, rs.num_channels if is_chn else 3)


def _views_forward(ctx, is_chn, what, settings_list, means3D, sh, colors_precomp, opacities, scales, rotations,
                   cov3Ds_precomp, expected_depth, antialiasing, features=None, bg_features=None):
    """Forward of _RasterizeGaussians (one view), _RasterizeGaussiansBatch and, with ``features``, _RasterizeJointBatch:
    (*colors, *radii[, *depths][, *feature images][, *expected depths, *alphas]), the depths for the rgbd variant (not
    ``is_chn``), the feature images with ``features``, the last two when ``expected_depth``."""
    joint = features is not None
    native, (R, color, radii, geom, binning, img, depth, exp_depth, alpha, *feat) = _forward(
        not is_chn, what, *_native_args(is_chn, joint, settings_list, means3D, sh, colors_precomp, opacities, scales,
                                        rotations, cov3Ds_precomp),
        want_exp_alpha=expected_depth, features=features, bg_features=bg_features, antialiasing=antialiasing)
    # the backward reuses the marshalled inputs; they also hold any contiguous copies their pointers refer to
    ctx.settings_list, ctx.R, ctx.native, ctx.expected_depth = settings_list, R, native, expected_depth
    ctx.is_chn, ctx.antialiasing = is_chn, antialiasing
    ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, sh, features, bg_features, *radii,
                          *geom, *binning, *img)
    ctx.mark_non_differentiable(*radii)
    outs = (*color, *radii)
    if not is_chn:
        ctx.mark_non_differentiable(*depth)  # no median-depth gradient in the reference (backward ignores it)
        outs += (*depth,)
    if joint:
        outs += (*feat[0],)
    if not (expected_depth or joint):
        return outs
    # gradients arrive as None for outputs the loss does not use: a loss on E / A alone runs no colour gradient
    # through the blend, one on the colours alone runs the plain backward, and a loss on one image of a joint render
    # leaves the other's gradient None
    ctx.set_materialize_grads(False)
    return outs + (*exp_depth, *alpha) if expected_depth else outs


def _camera_tensors(settings_list):
    """The camera tensors of the views, passed to the autograd functions as inputs so that they can receive
    gradients: viewmatrix, projmatrix, campos of each view in turn."""
    return [t for rs in settings_list for t in (rs.viewmatrix, rs.projmatrix, rs.campos)]


def _views_backward(ctx, what, saved, grad_outputs, cam_grad=False):
    """(per-view list of dL_dmeans2D, then the gradients of means3D, sh, colors_precomp, opacities, scales,
    rotations, cov3Ds_precomp[, features] summed over the views; None for an absent optional input), followed by the
    gradients of _camera_tensors(ctx.settings_list): computed with ``cam_grad``, else None.  ``saved`` is
    ctx.saved_tensors, ``grad_outputs`` the gradients of _views_forward's outputs."""
    V = len(ctx.settings_list)
    colors_precomp, means3D, scales, rotations, cov3Ds_precomp, sh, features, bg_features, *states = saved
    radii, geom, binning, img = states[:V], states[V:2 * V], states[2 * V:3 * V], states[3 * V:]
    rs = ctx.settings_list[0]
    H, W = rs.image_height, rs.image_width
    # without materialised gradients, an output the loss does not use has a None gradient: zeros
    fill = lambda gs, ch: [torch.zeros((ch, H, W), device=means3D.device) if g is None else g for g in gs]
    grad_colors = fill(grad_outputs[:V], rs.num_channels if ctx.is_chn else 3)
    k = (2 if ctx.is_chn else 3) * V  # past the colours, radii and depths
    g_feat = g_exp = g_alpha = None
    if features is not None:
        g_feat, k = fill(grad_outputs[k:k + V], features.size(1)), k + V
    if ctx.expected_depth:
        g_exp, g_alpha = grad_outputs[k:k + V], grad_outputs[k + V:k + 2 * V]
        g_exp = None if all(g is None for g in g_exp) else fill(g_exp, 1)
        g_alpha = None if all(g is None for g in g_alpha) else fill(g_alpha, 1)
    native = ctx.native
    if native is None:  # empty scene: the forward marshalled nothing
        native = _make_inputs(*_native_args(ctx.is_chn, features is not None, ctx.settings_list, means3D, sh,
                                            colors_precomp, means3D, scales, rotations, cov3Ds_precomp),
                              antialiasing=ctx.antialiasing)
    joint = None
    if features is not None:  # the table and background as the forward marshalled them (as given: empty scene)
        keep = native[2]
        joint = (keep.get("features", features), keep.get("bg_features", bg_features), g_feat)
    g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_sh, g_scales, g_rot, *tail = _backward(
        what, native, radii, grad_colors, geom, ctx.R, binning, img, g_exp, g_alpha, joint, cam_grad)
    g_features = tail[:1] if features is not None else []
    cams = _camera_tensors(ctx.settings_list)
    if cam_grad:
        # buffer order is the contiguous copy's, i.e. the tensor's own logical order (see _f32)
        g_cam = tail[-1]
        g_cams = [g_cam[i // 3, (0, 16, 32)[i % 3]:(16, 32, 35)[i % 3]].reshape(t.shape) for i, t in enumerate(cams)]
    else:
        g_cams = [None] * len(cams)

    def present(t, g):  # absent optional inputs were empty tensors; they get no gradient
        return g if t.numel() != 0 else None
    return (g_means2D, g_means3D, present(sh, g_sh), present(colors_precomp, g_colors), g_opac,
            present(scales, g_scales), present(rotations, g_rot), present(cov3Ds_precomp, g_cov3D), *g_features,
            *g_cams)


def make_module(variant: str):
    """Build (GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians,
    _RasterizeGaussians, _C) for variant 'chn' or 'rgbd'."""
    assert variant in ("chn", "rgbd")
    is_chn = variant == "chn"
    _C = _C_chn if is_chn else _C_rgbd

    if is_chn:
        class GaussianRasterizationSettings(NamedTuple):  # channel_rasterization/__init__.py:216-229
            image_height: int
            image_width: int
            tanfovx: float
            tanfovy: float
            bg: torch.Tensor
            scale_modifier: float
            viewmatrix: torch.Tensor
            projmatrix: torch.Tensor
            sh_degree: int
            campos: torch.Tensor
            prefiltered: bool
            debug: bool
            num_channels: int
    else:
        class GaussianRasterizationSettings(NamedTuple):  # rgbd_rasterization/__init__.py:159-171
            image_height: int
            image_width: int
            tanfovx: float
            tanfovy: float
            bg: torch.Tensor
            scale_modifier: float
            viewmatrix: torch.Tensor
            projmatrix: torch.Tensor
            sh_degree: int
            campos: torch.Tensor
            prefiltered: bool
            debug: bool

    class _RasterizeGaussians(torch.autograd.Function):
        @staticmethod
        def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                    raster_settings, expected_depth=False, antialiasing=False, *camera):
            # camera: _camera_tensors([raster_settings]), inputs only so that they can receive gradients
            rs = raster_settings
            try:
                return _views_forward(ctx, is_chn, "rasterize_gaussians", [rs], means3D, sh, colors_precomp, opacities,
                                      scales, rotations, cov3Ds_precomp, expected_depth, antialiasing)
            except Exception:
                if rs.debug:
                    args = [rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
                            cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height,
                            rs.image_width, sh, rs.sh_degree, rs.campos, rs.prefiltered]
                    _dump(args + [rs.debug, rs.num_channels] if is_chn else args, "snapshot_fw.dump")
                    print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise

        @staticmethod
        def backward(ctx, *grad_outputs):
            saved = ctx.saved_tensors
            try:
                g_means2D, g_means3D, *grads = _views_backward(ctx, "rasterize_gaussians_backward", saved,
                                                               grad_outputs, any(ctx.needs_input_grad[11:]))
            except Exception:
                rs = ctx.settings_list[0]
                if rs.debug:
                    colors_precomp, means3D, scales, rotations, cov3Ds_precomp, sh, _, _, radii, geom, binning, img = \
                        saved
                    args = [rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier,
                            cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_outputs[0], sh,
                            rs.sh_degree, rs.campos, geom, ctx.R[0], binning, img]
                    _dump(args + [rs.debug] if is_chn else args, "snapshot_bw.dump")
                    print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise
            *grads, g_view, g_proj, g_campos = grads
            return (g_means3D, g_means2D[0], *grads, None, None, None, g_view, g_proj, g_campos)

    def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                            raster_settings, *, expected_depth=False, antialiasing=False):
        """The reference's rasterize_gaussians; with ``expected_depth`` the outputs gain the expected depth
        E = sum_i w_i z_i and the accumulated opacity A = sum_i w_i, (1, H, W) each and differentiable (C <= 4).
        ``antialiasing``: 3DGS's opacity-compensated screen-space filter (INTEGRATION.md, "Anti-aliasing")."""
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                         cov3Ds_precomp, raster_settings, expected_depth, bool(antialiasing),
                                         *_camera_tensors([raster_settings]))

    class _RasterizeGaussiansBatch(torch.autograd.Function):
        """V views of the same Gaussians in one native call each way (the reference loops over
        single-view calls in Python, eval_segmentation.py:146-157).  Outputs per view are those of
        _RasterizeGaussians; the backward sums the per-Gaussian gradients over the views, the (P, C) feature
        gradient in place inside the kernels."""

        @staticmethod
        def forward(ctx, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings_list,
                    expected_depth, antialiasing, *means2D_camera):
            # means2D_camera: the V screen-space tensors, then _camera_tensors(settings_list)
            _check_batch_settings(settings_list)
            return _views_forward(ctx, is_chn, "rasterize_gaussians_batch", settings_list, means3D, sh, colors_precomp,
                                  opacities, scales, rotations, cov3Ds_precomp, expected_depth, antialiasing)

        @staticmethod
        def backward(ctx, *grad_outputs):
            V = len(ctx.settings_list)
            g_means2D, *grads = _views_backward(ctx, "rasterize_gaussians_backward_batch", ctx.saved_tensors,
                                                grad_outputs, any(ctx.needs_input_grad[10 + V:]))
            return (*grads[:-3 * V], None, None, None, *g_means2D, *grads[-3 * V:])

    def rasterize_gaussians_batch(means3D, means2D_list, opacities, settings_list, shs=None, colors_precomp=None,
                                  scales=None, rotations=None, cov3D_precomp=None, expected_depth=False,
                                  antialiasing=False):
        """Batched counterpart of GaussianRasterizer.forward: ``settings_list`` holds one
        GaussianRasterizationSettings per view (same image size / background tensor / channel count; only the
        cameras differ), ``means2D_list`` one screen-space tensor per view.  Returns a list of per-view tuples
        (color, radii[, depth][, expected depth, alpha]), the last two with ``expected_depth`` (see
        rasterize_gaussians, also for ``antialiasing``).  Batches larger than the native limit are split."""
        shs, colors_precomp, scales, rotations, cov3D_precomp = _optional_inputs(shs, colors_precomp, scales,
                                                                                 rotations, cov3D_precomp)
        results = []
        for lo in range(0, len(settings_list), _lib.MAX_BATCH):
            sl = list(settings_list[lo:lo + _lib.MAX_BATCH])
            m2 = list(means2D_list[lo:lo + _lib.MAX_BATCH])
            out = _RasterizeGaussiansBatch.apply(means3D, shs, colors_precomp, opacities, scales, rotations,
                                                 cov3D_precomp, sl, expected_depth, bool(antialiasing), *m2,
                                                 *_camera_tensors(sl))
            V = len(sl)
            per_view = 2 if is_chn else 3
            if expected_depth:
                per_view += 2
            for v in range(V):
                results.append(tuple(out[i * V + v] for i in range(per_view)))
        return results

    class GaussianRasterizer(nn.Module):  # channel_rasterization/__init__.py:232-289
        def __init__(self, raster_settings, antialiasing=False):
            """``antialiasing``: 3DGS's opacity-compensated screen-space filter for every render of this rasterizer
            (INTEGRATION.md, "Anti-aliasing"); not a settings field, whose layout is the reference's."""
            super().__init__()
            self.raster_settings = raster_settings
            self.antialiasing = bool(antialiasing)

        def markVisible(self, positions):
            with torch.no_grad():
                rs = self.raster_settings
                return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

        def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                    cov3D_precomp=None):
            shs, colors_precomp, scales, rotations, cov3D_precomp = _optional_inputs(shs, colors_precomp, scales,
                                                                                     rotations, cov3D_precomp)
            return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                       cov3D_precomp, self.raster_settings, antialiasing=self.antialiasing)

        def forward_expected_depth(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                                   rotations=None, cov3D_precomp=None):
            """forward() followed by the differentiable expected depth and alpha (see rasterize_gaussians)."""
            shs, colors_precomp, scales, rotations, cov3D_precomp = _optional_inputs(shs, colors_precomp, scales,
                                                                                     rotations, cov3D_precomp)
            return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                       cov3D_precomp, self.raster_settings, expected_depth=True,
                                       antialiasing=self.antialiasing)

    GaussianRasterizationSettings.__qualname__ = "GaussianRasterizationSettings"
    GaussianRasterizer.__qualname__ = "GaussianRasterizer"
    GaussianRasterizer.rasterize_batch = staticmethod(rasterize_gaussians_batch)
    return GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians, _RasterizeGaussians, _C


class _RasterizeJointBatch(torch.autograd.Function):
    """V views of the same Gaussians rendered twice from one geometry pass and one binning per view: the RGB image
    (with median depth, and expected depth / alpha when asked) and the image of a second colour table ``features``.
    Outputs: (*rgb, *radii, *depth, *feature images[, *expected depths, *alphas]).  The backward runs one geometry
    backward per view with the sum of both images' screen-space gradients."""

    @staticmethod
    def forward(ctx, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, features, bg_features,
                settings_list, expected_depth, antialiasing, *means2D_camera):
        # means2D_camera: the V screen-space tensors, then _camera_tensors(settings_list)
        _check_batch_settings(settings_list)
        return _views_forward(ctx, False, "rasterize_joint_batch", settings_list, means3D, sh, colors_precomp,
                              opacities, scales, rotations, cov3Ds_precomp, expected_depth, antialiasing, features,
                              bg_features)

    @staticmethod
    def backward(ctx, *grad_outputs):
        V = len(ctx.settings_list)
        g_means2D, *grads = _views_backward(ctx, "rasterize_joint_backward_batch", ctx.saved_tensors, grad_outputs,
                                            any(ctx.needs_input_grad[12 + V:]))
        return (*grads[:-3 * V], None, None, None, None, *g_means2D, *grads[-3 * V:])


def rasterize_joint_batch(means3D, means2D_list, opacities, settings_list, features, bg_features, shs=None,
                          colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None, expected_depth=False,
                          antialiasing=False):
    """The RGB-D rasterizer's rasterize_batch (``settings_list`` of rgbd GaussianRasterizationSettings, RGB colours
    from ``shs`` or ``colors_precomp``) that also renders ``features`` (P, c) over ``bg_features`` (c) from the same
    geometry and binning.  Returns a list of per-view tuples (rgb, radii, depth, feature image[, expected depth,
    alpha]).  ``means2D_list[v].grad`` receives the sum of both images' dL/dmean2D.  Batches larger than the native
    limit are split.  ``antialiasing`` as for rasterize_gaussians."""
    shs, colors_precomp, scales, rotations, cov3D_precomp = _optional_inputs(shs, colors_precomp, scales, rotations,
                                                                             cov3D_precomp)
    results = []
    per_view = 6 if expected_depth else 4
    for lo in range(0, len(settings_list), _lib.MAX_BATCH):
        sl = list(settings_list[lo:lo + _lib.MAX_BATCH])
        m2 = list(means2D_list[lo:lo + _lib.MAX_BATCH])
        out = _RasterizeJointBatch.apply(means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                         features, bg_features, sl, expected_depth, bool(antialiasing), *m2,
                                         *_camera_tensors(sl))
        V = len(sl)
        for v in range(V):
            results.append(tuple(out[i * V + v] for i in range(per_view)))
    return results
