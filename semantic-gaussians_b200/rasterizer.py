"""Autograd boundary of the rasterizer: the Python surface of the reference's two extensions
(``channel_rasterization/__init__.py`` and ``rgbd_rasterization/__init__.py``) over libsgb200.

``_C_chn`` / ``_C_rgbd`` reproduce the pybind entry points ``rasterize_gaussians``,
``rasterize_gaussians_backward`` and ``mark_visible`` (ext.cpp:16-18) with the reference's
positional argument lists and return tuples; ``make_module`` builds the
GaussianRasterizationSettings / GaussianRasterizer / _RasterizeGaussians trio for each variant.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


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


def _make_inputs(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                 viewmatrix, projmatrix, tan_fovx, tan_fovy, H, W, sh, degree, campos, prefiltered,
                 debug, num_channels):
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:61-64
    if not means3D.is_cuda:
        raise RuntimeError("means3D must be a CUDA tensor: the rasterizer has no CPU path")
    dev = means3D.device
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
        prefiltered=int(bool(prefiltered)), debug=int(bool(debug)))
    return inp, keep, dev


def _forward_impl(want_depth: bool, background, means3D, colors, opacity, scales, rotations, scale_modifier,
                  cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh,
                  degree, campos, prefiltered, debug, num_channels):
    lib = _lib.load()
    if means3D.ndimension() == 2 and means3D.size(0) == 0 and means3D.is_cuda:
        # Empty scene: the reference never enters the native forward (rasterize_points.cu:84) and
        # returns its zero-initialised outputs — zeros, not the background.
        dev = means3D.device
        z = torch.zeros((num_channels, image_height, image_width), dtype=torch.float32, device=dev)
        e8 = torch.empty((0,), dtype=torch.uint8, device=dev)
        radii = torch.zeros((0,), dtype=torch.int32, device=dev)
        img = torch.zeros((lib.sgb_image_bytes(image_width, image_height),), dtype=torch.uint8, device=dev)
        if want_depth:
            return 0, z, radii, e8, e8.clone(), img, torch.zeros((1, image_height, image_width), device=dev)
        return 0, z, radii, e8, e8.clone(), img
    inp, keep, dev = _make_inputs(background, means3D, colors, opacity, scales, rotations, scale_modifier,
                                  cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height,
                                  image_width, sh, degree, campos, prefiltered, debug, num_channels)
    P, H, W, Cn = inp.P, inp.H, inp.W, inp.C
    u8 = dict(dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        stream, ctx = _stream_ctx(dev)
        # every pixel / every radius is written by the kernels: no zero fill (the reference's
        # torch::full of out_color is pure waste, rasterize_points.cu:73)
        out_color = torch.empty((Cn, H, W), dtype=torch.float32, device=dev)
        out_depth = torch.empty((1, H, W), dtype=torch.float32, device=dev) if want_depth else None
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        geom = torch.empty((lib.sgb_geometry_bytes(P),), **u8)
        img = torch.empty((lib.sgb_image_bytes(W, H),), **u8)
        R = C.c_int64(0)
        _lib.check(lib.sgb_forward_geometry(ctx, C.byref(inp), geom.data_ptr(), radii.data_ptr(), C.byref(R),
                                            stream), "rasterize_gaussians (geometry)")
        binning = torch.empty((lib.sgb_binning_bytes(R.value),), **u8)
        _lib.check(lib.sgb_forward_render(ctx, C.byref(inp), R.value, geom.data_ptr(), binning.data_ptr(),
                                          img.data_ptr(), radii.data_ptr(), out_color.data_ptr(),
                                          _ptr(out_depth), stream), "rasterize_gaussians (render)")
    del keep
    if want_depth:
        return int(R.value), out_color, radii, geom, binning, img, out_depth
    return int(R.value), out_color, radii, geom, binning, img


def _backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                   viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos, geomBuffer,
                   R, binningBuffer, imageBuffer, debug, opacities_placeholder=None):
    lib = _lib.load()
    Cn, H, W = dL_dout_color.shape  # rasterize_points.cu:146-148
    dev = means3D.device
    P = means3D.size(0)
    # opacities are not an input of Rasterizer::backward (they live in the geometry state); the
    # struct field only has to be non-null for validation.
    opac = opacities_placeholder if opacities_placeholder is not None else means3D
    inp, keep, dev = _make_inputs(background, means3D, colors, opac, scales, rotations, scale_modifier,
                                  cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, H, W, sh, degree,
                                  campos, False, debug, Cn)
    M = inp.M
    z = dict(dtype=torch.float32, device=dev)
    dL_dmeans3D = torch.zeros((P, 3), **z)
    dL_dmeans2D = torch.zeros((P, 3), **z)
    dL_dcolors = torch.zeros((P, Cn), **z)
    dL_dconic = torch.zeros((P, 2, 2), **z)
    dL_dopacity = torch.zeros((P, 1), **z)
    dL_dcov3D = torch.zeros((P, 6), **z)
    dL_dsh = torch.zeros((P, M, 3), **z)
    dL_dscales = torch.zeros((P, 3), **z)
    dL_drotations = torch.zeros((P, 4), **z)
    gout = _f32(dL_dout_color, dev, "dL_dout_color")
    grads = _lib.ViewGrads(
        dL_dmeans2D=dL_dmeans2D.data_ptr(), dL_dconic=dL_dconic.data_ptr(), dL_dopacity=dL_dopacity.data_ptr(),
        dL_dcolors=dL_dcolors.data_ptr(), dL_dmeans3D=dL_dmeans3D.data_ptr(), dL_dcov3D=dL_dcov3D.data_ptr(),
        dL_dsh=dL_dsh.data_ptr() if M > 0 else None, dL_dscales=dL_dscales.data_ptr(),
        dL_drotations=dL_drotations.data_ptr())
    if P != 0:
        with torch.cuda.device(dev):
            stream, ctx = _stream_ctx(dev)
            _lib.check(lib.sgb_backward(ctx, C.byref(inp), int(R), radii.data_ptr(), geomBuffer.data_ptr(),
                                        binningBuffer.data_ptr(), imageBuffer.data_ptr(), gout.data_ptr(),
                                        C.byref(grads), stream), "rasterize_gaussians_backward")
    del keep
    return dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations


# ------------------------------------------------------------------------------------------------ batched views
def _ptr_array(ptrs):
    arr = (C.c_void_p * len(ptrs))()
    for i, p in enumerate(ptrs):
        arr[i] = p
    return arr


def _camera_array(settings_list, dev, keep):
    cams = (_lib.Camera * len(settings_list))()
    for i, rs in enumerate(settings_list):
        v, p, c = _f32(rs.viewmatrix, dev, "viewmatrix"), _f32(rs.projmatrix, dev, "projmatrix"), _f32(rs.campos, dev, "campos")
        keep += [v, p, c]
        cams[i] = _lib.Camera(viewmatrix=v.data_ptr(), projmatrix=p.data_ptr(), campos=c.data_ptr(),
                              tan_fovx=float(rs.tanfovx), tan_fovy=float(rs.tanfovy))
    return cams


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
    return rs0


def _forward_batch_impl(want_depth: bool, settings_list, means3D, colors, opacity, scales, rotations, cov3D_precomp,
                        sh, num_channels):
    """V views of the same Gaussians through sgb_forward_geometry_batch / sgb_forward_render_batch: one stream
    sync for all instance counts, one for all weight-pool checks.  Returns per-view lists."""
    lib = _lib.load()
    rs0 = _check_batch_settings(settings_list)
    V = len(settings_list)
    inp, keep, dev = _make_inputs(rs0.bg, means3D, colors, opacity, scales, rotations, rs0.scale_modifier,
                                  cov3D_precomp, rs0.viewmatrix, rs0.projmatrix, rs0.tanfovx, rs0.tanfovy,
                                  rs0.image_height, rs0.image_width, sh, rs0.sh_degree, rs0.campos, rs0.prefiltered,
                                  getattr(rs0, "debug", False), num_channels)
    P, H, W, Cn = inp.P, inp.H, inp.W, inp.C
    if P == 0:
        raise ValueError("batched rasterization of an empty scene: use the single-view call")
    u8 = dict(dtype=torch.uint8, device=dev)
    keep_list = [keep]
    with torch.cuda.device(dev):
        stream, ctx = _stream_ctx(dev)
        cams = _camera_array(settings_list, dev, keep_list)
        out_color = [torch.empty((Cn, H, W), dtype=torch.float32, device=dev) for _ in range(V)]
        out_depth = [torch.empty((1, H, W), dtype=torch.float32, device=dev) for _ in range(V)] if want_depth else None
        radii = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(V)]
        geom = [torch.empty((lib.sgb_geometry_bytes(P),), **u8) for _ in range(V)]
        img = [torch.empty((lib.sgb_image_bytes(W, H),), **u8) for _ in range(V)]
        R = (C.c_int64 * V)()
        _lib.check(lib.sgb_forward_geometry_batch(ctx, C.byref(inp), V, cams, _ptr_array([g.data_ptr() for g in geom]),
                                                  _ptr_array([r.data_ptr() for r in radii]), R, stream),
                   "rasterize_gaussians_batch (geometry)")
        binning = [torch.empty((lib.sgb_binning_bytes(R[v]),), **u8) for v in range(V)]
        _lib.check(lib.sgb_forward_render_batch(
            ctx, C.byref(inp), V, cams, R, _ptr_array([g.data_ptr() for g in geom]),
            _ptr_array([b.data_ptr() for b in binning]), _ptr_array([i.data_ptr() for i in img]),
            _ptr_array([r.data_ptr() for r in radii]), _ptr_array([o.data_ptr() for o in out_color]),
            _ptr_array([d.data_ptr() for d in out_depth]) if want_depth else None, stream),
            "rasterize_gaussians_batch (render)")
    del keep_list
    return [int(R[v]) for v in range(V)], out_color, radii, geom, binning, img, out_depth


def _backward_batch_impl(settings_list, means3D, radii, colors, scales, rotations, cov3D_precomp, dL_dout, sh,
                         geom, R, binning, img, num_channels):
    """sgb_backward_batch: the (P, C) colour / feature gradient accumulates over the views in ONE buffer; the small
    per-Gaussian gradients are per view and summed here (means2D stays per view)."""
    lib = _lib.load()
    rs0 = settings_list[0]
    V = len(settings_list)
    H, W = rs0.image_height, rs0.image_width
    inp, keep, dev = _make_inputs(rs0.bg, means3D, colors, means3D, scales, rotations, rs0.scale_modifier,
                                  cov3D_precomp, rs0.viewmatrix, rs0.projmatrix, rs0.tanfovx, rs0.tanfovy, H, W, sh,
                                  rs0.sh_degree, rs0.campos, False, getattr(rs0, "debug", False), num_channels)
    P, M, Cn = inp.P, inp.M, inp.C
    z = dict(dtype=torch.float32, device=dev)
    # precomputed colours / features: ONE (P, C) buffer, summed over the views in place.  SH path: the per-view RGB
    # gradient is an input of that view's SH backward (backward.cu:385-386), so every view needs its own (P, 3).
    shared = M == 0
    dL_dcolors = torch.zeros((P, Cn) if shared else (V, P, Cn), **z)
    per = dict(dL_dmeans3D=(P, 3), dL_dmeans2D=(P, 3), dL_dconic=(P, 2, 2), dL_dopacity=(P, 1), dL_dcov3D=(P, 6),
               dL_dsh=(P, M, 3), dL_dscales=(P, 3), dL_drotations=(P, 4))
    small = {k: torch.zeros((V,) + shp, **z) for k, shp in per.items()}
    gouts = [_f32(g, dev, "dL_dout_color") for g in dL_dout]
    grads = (_lib.ViewGrads * V)()
    for v in range(V):
        grads[v] = _lib.ViewGrads(
            dL_dmeans2D=small["dL_dmeans2D"][v].data_ptr(), dL_dconic=small["dL_dconic"][v].data_ptr(),
            dL_dopacity=small["dL_dopacity"][v].data_ptr(),
            dL_dcolors=(dL_dcolors if shared else dL_dcolors[v]).data_ptr(),
            dL_dmeans3D=small["dL_dmeans3D"][v].data_ptr(), dL_dcov3D=small["dL_dcov3D"][v].data_ptr(),
            dL_dsh=small["dL_dsh"][v].data_ptr() if M > 0 else None, dL_dscales=small["dL_dscales"][v].data_ptr(),
            dL_drotations=small["dL_drotations"][v].data_ptr())
    keep_list = [keep]
    with torch.cuda.device(dev):
        stream, ctx = _stream_ctx(dev)
        cams = _camera_array(settings_list, dev, keep_list)
        Rarr = (C.c_int64 * V)(*[int(r) for r in R])
        _lib.check(lib.sgb_backward_batch(
            ctx, C.byref(inp), V, cams, Rarr, _ptr_array([r.data_ptr() for r in radii]),
            _ptr_array([g.data_ptr() for g in geom]), _ptr_array([b.data_ptr() for b in binning]),
            _ptr_array([i.data_ptr() for i in img]), _ptr_array([g.data_ptr() for g in gouts]), grads, stream),
            "rasterize_gaussians_backward_batch")
    del keep_list
    if not shared:
        dL_dcolors = dL_dcolors.sum(0)
    return (small["dL_dmeans2D"], dL_dcolors, small["dL_dopacity"].sum(0), small["dL_dmeans3D"].sum(0),
            small["dL_dcov3D"].sum(0), small["dL_dsh"].sum(0), small["dL_dscales"].sum(0),
            small["dL_drotations"].sum(0))


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


class _C_chn:
    """pybind surface of channel_rasterization._C (rasterize_points.cu:38-223, ext.cpp:16-18)."""

    @staticmethod
    def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                            viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree,
                            campos, prefiltered, debug, num_channels):
        return _forward_impl(False, background, means3D, colors, opacity, scales, rotations, scale_modifier,
                             cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width,
                             sh, degree, campos, prefiltered, debug, num_channels)

    @staticmethod
    def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh,
                                     degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug):
        return _backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                              viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos,
                              geomBuffer, R, binningBuffer, imageBuffer, debug)

    mark_visible = staticmethod(_mark_visible)


class _C_rgbd:
    """pybind surface of rgbd_rasterization._C (18 / 20 arguments, forward also returns depth)."""

    @staticmethod
    def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                            viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree,
                            campos, prefiltered):
        return _forward_impl(True, background, means3D, colors, opacity, scales, rotations, scale_modifier,
                             cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width,
                             sh, degree, campos, prefiltered, False, 3)

    @staticmethod
    def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh,
                                     degree, campos, geomBuffer, R, binningBuffer, imageBuffer):
        return _backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                              viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos,
                              geomBuffer, R, binningBuffer, imageBuffer, False)

    mark_visible = staticmethod(_mark_visible)


def _dump(args, path):
    """Reference debug behaviour without its unconditional CPU deep copy: the argument snapshot is
    taken only when the native call has already failed (channel_rasterization/__init__.py:86-100)."""
    try:
        torch.save(tuple(a.detach().cpu() if isinstance(a, torch.Tensor) else a for a in args), path)
    except Exception:  # pragma: no cover - best effort
        pass


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
                    raster_settings):
            rs = raster_settings
            args = [rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
                    cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height,
                    rs.image_width, sh, rs.sh_degree, rs.campos, rs.prefiltered]
            if is_chn:
                args += [rs.debug, rs.num_channels]
            try:
                out = _C.rasterize_gaussians(*args)
            except Exception:
                if rs.debug:
                    _dump(args, "snapshot_fw.dump")
                    print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise
            if is_chn:
                num_rendered, color, radii, geomBuffer, binningBuffer, imgBuffer = out
                depth = None
            else:
                num_rendered, color, radii, geomBuffer, binningBuffer, imgBuffer, depth = out
            ctx.raster_settings = rs
            ctx.num_rendered = num_rendered
            ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
                                  binningBuffer, imgBuffer)
            ctx.mark_non_differentiable(radii)
            if is_chn:
                return color, radii
            ctx.mark_non_differentiable(depth)  # no depth gradient in the reference (backward ignores it)
            return color, radii, depth

        @staticmethod
        def backward(ctx, grad_out_color, *_unused):
            rs = ctx.raster_settings
            (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer,
             imgBuffer) = ctx.saved_tensors
            args = [rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                    rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_out_color, sh, rs.sh_degree, rs.campos,
                    geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer]
            if is_chn:
                args.append(rs.debug)
            try:
                (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh,
                 grad_scales, grad_rotations) = _C.rasterize_gaussians_backward(*args)
            except Exception:
                if rs.debug:
                    _dump(args, "snapshot_bw.dump")
                    print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise

            def present(t, g):  # absent optional inputs were empty tensors; they get no gradient
                return g if t.numel() != 0 else None
            return (grad_means3D, grad_means2D, present(sh, grad_sh), present(colors_precomp, grad_colors_precomp),
                    grad_opacities, present(scales, grad_scales), present(rotations, grad_rotations),
                    present(cov3Ds_precomp, grad_cov3Ds_precomp), None)

    def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                            raster_settings):
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                         cov3Ds_precomp, raster_settings)

    class _RasterizeGaussiansBatch(torch.autograd.Function):
        """V views of the same Gaussians in one native call each way (the reference loops over
        single-view calls in Python, eval_segmentation.py:146-157).  Outputs per view are those of
        _RasterizeGaussians; the backward sums the per-Gaussian gradients over the views, the (P, C) feature
        gradient in place inside the kernels."""

        @staticmethod
        def forward(ctx, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings_list,
                    *means2D):
            V = len(settings_list)
            nch = settings_list[0].num_channels if is_chn else 3
            R, color, radii, geom, binning, img, depth = _forward_batch_impl(
                not is_chn, settings_list, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh, nch)
            ctx.settings_list, ctx.R, ctx.V, ctx.nch = list(settings_list), R, V, nch
            ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, sh, *radii, *geom,
                                  *binning, *img)
            ctx.mark_non_differentiable(*radii)
            if is_chn:
                return (*color, *radii)
            ctx.mark_non_differentiable(*depth)
            return (*color, *radii, *depth)

        @staticmethod
        def backward(ctx, *grad_outputs):
            V = ctx.V
            saved = ctx.saved_tensors
            colors_precomp, means3D, scales, rotations, cov3Ds_precomp, sh = saved[:6]
            rest = saved[6:]
            radii, geom, binning, img = rest[:V], rest[V:2 * V], rest[2 * V:3 * V], rest[3 * V:4 * V]
            rs0 = ctx.settings_list[0]
            gouts = []
            for v in range(V):
                g = grad_outputs[v]
                if g is None:
                    g = torch.zeros((ctx.nch, rs0.image_height, rs0.image_width), dtype=torch.float32,
                                    device=means3D.device)
                gouts.append(g)
            (g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_sh, g_scales, g_rot) = _backward_batch_impl(
                ctx.settings_list, means3D, radii, colors_precomp, scales, rotations, cov3Ds_precomp, gouts, sh, geom,
                ctx.R, binning, img, ctx.nch)

            def present(t, g):
                return g if t.numel() != 0 else None
            return (g_means3D, present(sh, g_sh), present(colors_precomp, g_colors), g_opac, present(scales, g_scales),
                    present(rotations, g_rot), present(cov3Ds_precomp, g_cov3D), None,
                    *[g_means2D[v] for v in range(V)])

    def rasterize_gaussians_batch(means3D, means2D_list, opacities, settings_list, shs=None, colors_precomp=None,
                                  scales=None, rotations=None, cov3D_precomp=None):
        """Batched counterpart of GaussianRasterizer.forward: ``settings_list`` holds one
        GaussianRasterizationSettings per view (same image size / background tensor / channel count; only the
        cameras differ), ``means2D_list`` one screen-space tensor per view.  Returns a list of per-view tuples
        (color, radii[, depth]).  Batches larger than the native limit are split."""
        if (shs is None) == (colors_precomp is None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
                (scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        empty = torch.Tensor([])
        e = lambda t: empty if t is None else t
        results = []
        for lo in range(0, len(settings_list), _lib.MAX_BATCH):
            sl = list(settings_list[lo:lo + _lib.MAX_BATCH])
            m2 = list(means2D_list[lo:lo + _lib.MAX_BATCH])
            out = _RasterizeGaussiansBatch.apply(means3D, e(shs), e(colors_precomp), opacities, e(scales), e(rotations),
                                                 e(cov3D_precomp), sl, *m2)
            V = len(sl)
            for v in range(V):
                results.append((out[v], out[V + v]) if is_chn else (out[v], out[V + v], out[2 * V + v]))
        return results

    class GaussianRasterizer(nn.Module):  # channel_rasterization/__init__.py:232-289
        def __init__(self, raster_settings):
            super().__init__()
            self.raster_settings = raster_settings

        def markVisible(self, positions):
            with torch.no_grad():
                rs = self.raster_settings
                return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

        def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                    cov3D_precomp=None):
            rs = self.raster_settings
            if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
                raise Exception("Please provide excatly one of either SHs or precomputed colors!")
            if ((scales is None or rotations is None) and cov3D_precomp is None) or (
                    (scales is not None or rotations is not None) and cov3D_precomp is not None):
                raise Exception(
                    "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
            empty = torch.Tensor([])
            shs = empty if shs is None else shs
            colors_precomp = empty if colors_precomp is None else colors_precomp
            scales = empty if scales is None else scales
            rotations = empty if rotations is None else rotations
            cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp
            return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                       cov3D_precomp, rs)

    GaussianRasterizationSettings.__qualname__ = "GaussianRasterizationSettings"
    GaussianRasterizer.__qualname__ = "GaussianRasterizer"
    GaussianRasterizer.rasterize_batch = staticmethod(rasterize_gaussians_batch)
    return GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians, _RasterizeGaussians, _C
