"""render() / render_chn(): the reference's Render API (model/renderer.py:20-130 and :134-246) over
the H100 rasterizer.  Signatures, argument semantics and returned dict keys are the reference's;
``pc`` is any object with the GaussianModel getters the reference reads (get_xyz, get_opacity,
get_scaling, get_rotation, get_features, get_covariance[_rotation], active_sh_degree,
max_sh_degree) and ``pipe`` any object with convert_shs_python / compute_cov3d_python / debug.

Differences from the reference, all on purpose:
  * tensors are created on ``pc.get_xyz.device`` instead of the literal "cuda";
  * render_chn() honours ``pipe.debug`` instead of hard-coding debug=True
    (model/renderer.py:181), which made every call deep-copy all inputs to the CPU.

Addition: render_with_depth() (render()'s parameters; render() keeps the reference's exact signature) and
render_batch(..., differentiable_depth=True) also return, from the same pass,
  "expected_depth"  E = sum_i w_i z_i  (1, H, W)   w_i = alpha_i T_i, z_i the view-space depth of Gaussian i
  "alpha"           A = sum_i w_i      (1, H, W)
with gradients (to means3D through z and through the blend weights, to opacity, scales / rotations or cov3D, and
the screen-space points).  No background term: the normalised depth is E / A.clamp_min(eps).  "depth" stays the
reference's non-differentiable median depth.

Addition: ``pipe.antialiasing`` (3DGS's PipelineParams attribute; absent means False) turns on the opacity-compensated
screen-space filter in every render here: each Gaussian's opacity is scaled by sqrt(det C0 / det C), C0 its screen
covariance before the fixed 0.3 px² dilation and C after it, so a Gaussian covers the same area at every image size.
Radii, tiles and binning are unchanged.  Train and render a model with the same setting (INTEGRATION.md).

Addition: render_with_features() / render_with_features_batch() train colour and a per-Gaussian feature field
together: one geometry pass and one binning per view produce render()'s dict (plus "expected_depth" / "alpha" under
``differentiable_depth``) and "features" (c, H, W), the image of a (P, c) table over its background, bitwise what
render() and render_chn() give.  One backward carries both losses.  ``viewspace_points.grad`` holds the sum of both
images' screen-space gradients, so the densification statistic (add_densification_stats) sees the feature loss too.
"""
import math
from functools import partial

import torch

from . import channel_rasterization as chn_rasterize
from .rasterizer import rasterize_joint_batch
from .rgbd_rasterization import GaussianRasterizationSettings, GaussianRasterizer
from .sh_utils import eval_sh


def _antialiasing(pipe) -> bool:
    return bool(getattr(pipe, "antialiasing", False))


def _prepare(viewpoint_camera, pc, pipe, scaling_modifier, override_color, override_shape, foreground, world_rotate):
    xyz = pc.get_xyz
    # zero tensor whose .grad receives the screen-space mean gradients (model/renderer.py:36-41)
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    tanfovx = math.tan(viewpoint_camera.FoVx * 0.5)
    tanfovy = math.tan(viewpoint_camera.FoVy * 0.5)
    if override_shape is not None:
        image_height, image_width = override_shape[1], override_shape[0]
    else:
        image_height, image_width = int(viewpoint_camera.image_height), int(viewpoint_camera.image_width)

    means3D = xyz
    opacity = pc.get_opacity
    if foreground is not None:
        opacity[~foreground] = 0  # model/renderer.py:74-75

    scales = rotations = cov3D_precomp = None
    if pipe.compute_cov3d_python:
        cov3D_precomp = pc.get_covariance(scaling_modifier)
    else:
        scales, rotations = pc.get_scaling, pc.get_rotation
    if world_rotate is not None:  # model/renderer.py:88-93
        scales = rotations = None
        world_rotate = torch.from_numpy(world_rotate).float().to(xyz.device)
        means3D = means3D @ world_rotate
        cov3D_precomp = pc.get_covariance_rotation(scaling_modifier, world_rotate)

    shs = colors_precomp = None
    if override_color is None:
        if pipe.convert_shs_python:  # model/renderer.py:100-105
            shs_view = pc.get_features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
            dir_pp = pc.get_xyz - viewpoint_camera.camera_center.repeat(pc.get_features.shape[0], 1)
            dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
            sh2rgb = eval_sh(pc.active_sh_degree, shs_view, dir_pp_normalized)
            colors_precomp = torch.clamp_min(sh2rgb + 0.5, 0.0)
        else:
            shs = pc.get_features
    else:
        colors_precomp = override_color
    common = dict(image_height=image_height, image_width=image_width, tanfovx=tanfovx, tanfovy=tanfovy,
                  scale_modifier=scaling_modifier, viewmatrix=viewpoint_camera.world_view_transform,
                  projmatrix=viewpoint_camera.full_proj_transform, sh_degree=pc.active_sh_degree,
                  campos=viewpoint_camera.camera_center, prefiltered=False)
    call = dict(means3D=means3D, means2D=screenspace_points, shs=shs, colors_precomp=colors_precomp,
                opacities=opacity, scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
    return screenspace_points, common, call


def _prepare_views(cameras, pc, pipe, scaling_modifier, override_color, override_shape, foreground, world_rotate,
                   make_settings):
    """_prepare for a batch of cameras: the Gaussian-side tensors are prepared ONCE (the reference's per-view loop,
    eval_segmentation.py:146-157 / fusion.py:106-120, re-evaluates the activations for every view).  Returns the
    rasterizer settings of every camera (``make_settings(**common)`` with the camera's fields), its screen-space
    points (camera 0's from _prepare, the others new zero tensors like them) and the call arguments."""
    pts0, common0, call = _prepare(cameras[0], pc, pipe, scaling_modifier, override_color, override_shape, foreground,
                                   world_rotate)
    settings, points = [], []
    for i, cam in enumerate(cameras):
        common = dict(common0, tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
                      viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center)
        if override_shape is None and (int(cam.image_height), int(cam.image_width)) != (common0["image_height"],
                                                                                        common0["image_width"]):
            raise ValueError("the views of a batch must share the image size")
        settings.append(make_settings(**common))
        if i == 0:
            points.append(pts0)
        else:
            p = torch.zeros_like(pts0, requires_grad=True) + 0
            try:
                p.retain_grad()
            except Exception:
                pass
            points.append(p)
    return settings, points, call


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
           override_shape=None, foreground=None, world_rotate=None):
    """RGB + median depth (rgbd rasterizer).  Background tensor (bg_color) must be on the GPU."""
    return _render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, override_shape, foreground,
                   world_rotate, False)


def render_with_depth(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
                      override_shape=None, foreground=None, world_rotate=None):
    """render()'s dict plus the differentiable "expected_depth" and "alpha" of the same pass (module docstring)."""
    return _render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, override_shape, foreground,
                   world_rotate, True)


def _render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, override_shape, foreground,
            world_rotate, differentiable_depth):
    screenspace_points, common, call = _prepare(viewpoint_camera, pc, pipe, scaling_modifier, override_color,
                                                override_shape, foreground, world_rotate)
    raster_settings = GaussianRasterizationSettings(bg=bg_color, debug=pipe.debug, **common)
    rasterizer = GaussianRasterizer(raster_settings=raster_settings, antialiasing=_antialiasing(pipe))
    if differentiable_depth:
        rendered_image, radii, depth, exp_depth, alpha = rasterizer.forward_expected_depth(**call)
    else:
        rendered_image, radii, depth = rasterizer(**call)
    out = {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
           "radii": radii, "depth": depth}
    if differentiable_depth:
        out.update(expected_depth=exp_depth, alpha=alpha)
    return out


def render_chn(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, num_channels=3,
               override_color=None, override_shape=None, foreground=None, world_rotate=None):
    """C-channel feature raster (channel rasterizer)."""
    screenspace_points, common, call = _prepare(viewpoint_camera, pc, pipe, scaling_modifier, override_color,
                                                override_shape, foreground, world_rotate)
    raster_settings = chn_rasterize.GaussianRasterizationSettings(
        bg=bg_color, debug=bool(getattr(pipe, "debug", False)), num_channels=num_channels, **common)
    rasterizer = chn_rasterize.GaussianRasterizer(raster_settings=raster_settings, antialiasing=_antialiasing(pipe))
    rendered_image, radii = rasterizer.forward(**call)
    return {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
            "radii": radii}


def _render_batch(variant, cameras, pc, pipe, bg_color, scaling_modifier, num_channels, override_color, override_shape,
                  foreground, world_rotate, differentiable_depth=False):
    """Shared body of render_batch / render_chn_batch: the views go through _prepare_views and the batched native
    calls (rasterizer.rasterize_gaussians_batch)."""
    cameras = list(cameras)
    if not cameras:
        return []
    single = (render_with_depth if differentiable_depth else render) if variant == "rgbd" else (
        lambda cam, *a, **k: render_chn(cam, *a, num_channels=num_channels, **k))
    per_view_colors = override_color is None and pipe.convert_shs_python   # python SH -> colours depend on the camera
    if per_view_colors:
        return [single(cam, pc, pipe, bg_color, scaling_modifier=scaling_modifier, override_color=override_color,
                       override_shape=override_shape, foreground=foreground, world_rotate=world_rotate)
                for cam in cameras]
    if variant == "chn":
        make_settings = partial(chn_rasterize.GaussianRasterizationSettings, bg=bg_color,
                                debug=bool(getattr(pipe, "debug", False)), num_channels=num_channels)
        Rast = chn_rasterize.GaussianRasterizer
    else:
        make_settings = partial(GaussianRasterizationSettings, bg=bg_color, debug=pipe.debug)
        Rast = GaussianRasterizer
    settings, points, call = _prepare_views(cameras, pc, pipe, scaling_modifier, override_color, override_shape,
                                            foreground, world_rotate, make_settings)
    outs = Rast.rasterize_batch(call["means3D"], points, call["opacities"], settings, shs=call["shs"],
                                colors_precomp=call["colors_precomp"], scales=call["scales"],
                                rotations=call["rotations"], cov3D_precomp=call["cov3D_precomp"],
                                expected_depth=differentiable_depth, antialiasing=_antialiasing(pipe))
    res = []
    for pts, o in zip(points, outs):
        d = {"render": o[0], "viewspace_points": pts, "visibility_filter": o[1] > 0, "radii": o[1]}
        if variant == "rgbd":
            d["depth"] = o[2]
        if differentiable_depth:
            d.update(expected_depth=o[3], alpha=o[4])
        res.append(d)
    return res


def render_batch(cameras, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
                 override_shape=None, foreground=None, world_rotate=None, *, differentiable_depth=False):
    """``[render(cam, ...) for cam in cameras]`` through the batched native path: same per-view dicts."""
    return _render_batch("rgbd", cameras, pc, pipe, bg_color, scaling_modifier, 3, override_color, override_shape,
                         foreground, world_rotate, differentiable_depth)


def render_chn_batch(cameras, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, num_channels=3,
                     override_color=None, override_shape=None, foreground=None, world_rotate=None):
    """``[render_chn(cam, ...) for cam in cameras]`` through the batched native path (BASELINE config K4: a rank's
    share of a view batch).  Backward of any loss over the returned images sums the per-Gaussian gradients over the
    views inside the kernels — one (P, C) feature-gradient buffer for the whole batch."""
    return _render_batch("chn", cameras, pc, pipe, bg_color, scaling_modifier, num_channels, override_color,
                         override_shape, foreground, world_rotate)


def render_with_features(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, features: torch.Tensor,
                         bg_features: torch.Tensor, scaling_modifier=1.0, override_color=None, override_shape=None,
                         foreground=None, world_rotate=None, *, differentiable_depth=False):
    """render()'s dict (render_with_depth()'s under ``differentiable_depth``) plus "features" (c, H, W): the image of
    ``features`` (P, c) over ``bg_features`` (c), from the same geometry pass and binning as the RGB image.  Gradients
    reach ``features``, the Gaussian parameters and ``viewspace_points`` from both images (module docstring)."""
    return render_with_features_batch([viewpoint_camera], pc, pipe, bg_color, features, bg_features,
                                      scaling_modifier=scaling_modifier, override_color=override_color,
                                      override_shape=override_shape, foreground=foreground, world_rotate=world_rotate,
                                      differentiable_depth=differentiable_depth)[0]


def render_with_features_batch(cameras, pc, pipe, bg_color: torch.Tensor, features: torch.Tensor,
                               bg_features: torch.Tensor, scaling_modifier=1.0, override_color=None,
                               override_shape=None, foreground=None, world_rotate=None, *, differentiable_depth=False):
    """``[render_with_features(cam, ...) for cam in cameras]`` through the batched native calls, split at the native
    batch limit as render_batch is."""
    cameras = list(cameras)
    if not cameras:
        return []
    if override_color is None and pipe.convert_shs_python:  # python SH -> colours depend on the camera
        groups = [[cam] for cam in cameras]
    else:
        groups = [cameras]
    res = []
    for group in groups:
        settings, points, call = _prepare_views(group, pc, pipe, scaling_modifier, override_color, override_shape,
                                                foreground, world_rotate,
                                                partial(GaussianRasterizationSettings, bg=bg_color, debug=pipe.debug))
        outs = rasterize_joint_batch(call["means3D"], points, call["opacities"], settings, features, bg_features,
                                     shs=call["shs"], colors_precomp=call["colors_precomp"], scales=call["scales"],
                                     rotations=call["rotations"], cov3D_precomp=call["cov3D_precomp"],
                                     expected_depth=differentiable_depth, antialiasing=_antialiasing(pipe))
        for pts, o in zip(points, outs):
            d = {"render": o[0], "viewspace_points": pts, "visibility_filter": o[1] > 0, "radii": o[1],
                 "depth": o[2], "features": o[3]}
            if differentiable_depth:
                d.update(expected_depth=o[4], alpha=o[5])
            res.append(d)
    return res
