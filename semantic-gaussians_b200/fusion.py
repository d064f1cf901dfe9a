"""2D-feature → 3D-Gaussian fusion on the GPU: drop-in for the reference's
``PointCloudToImageMapper`` (dataset/fusion_utils.py:17-78) and the per-view accumulate loop of
``fuse_one_scene`` (fusion.py:57-148), backed by libsgb200's fusion kernels."""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Union

import numpy as np
import torch

from . import _lib

ArrayLike = Union[np.ndarray, torch.Tensor]


def _dev_tensor(a: ArrayLike, dtype, device) -> torch.Tensor:
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(device)


class PointCloudToImageMapper(object):
    """Same constructor, attributes and ``compute_mapping`` contract as the reference class."""

    def __init__(self, image_dim, visibility_threshold=0.25, cut_bound=0, intrinsics=None, device="cuda"):
        self.image_dim = image_dim
        self.vis_thres = visibility_threshold
        self.cut_bound = cut_bound
        self.device = torch.device(device)
        # fusion_utils.py:22-28: rescale the intrinsics to image_dim
        self.intrinsics = np.array(intrinsics, dtype=np.float64).copy()
        scale_x = self.image_dim[0] / (self.intrinsics[0, 2] * 2)
        scale_y = self.image_dim[1] / (self.intrinsics[1, 2] * 2)
        self.intrinsics[0, 0] *= scale_x
        self.intrinsics[1, 1] *= scale_y
        self.intrinsics[0, 2] = self.image_dim[0] / 2
        self.intrinsics[1, 2] = self.image_dim[1] / 2

    # -- native view descriptor ---------------------------------------------------------------
    def _view(self, world_to_camera: ArrayLike, coords: ArrayLike, depth, keep: list) -> _lib.FusionView:
        dev = self.device
        xyz = _dev_tensor(coords, torch.float32, dev)
        w2c = _dev_tensor(world_to_camera, torch.float32, dev)
        if xyz.ndim != 2 or xyz.shape[1] != 3:
            raise ValueError("coords must be (N, 3)")
        if tuple(w2c.shape) != (4, 4):
            raise ValueError("world_to_camera must be 4x4")
        keep += [xyz, w2c]
        mode, dptr = _lib.DEPTH_NONE, None
        if isinstance(depth, str):  # fusion_utils.py:57: any string means "surface"
            mode = _lib.DEPTH_SURFACE
        elif depth is not None:
            if isinstance(depth, torch.Tensor):
                d = depth
                if d.dtype not in (torch.float32, torch.float64):
                    d = d.double()
            else:
                d = np.asarray(depth)
                if d.dtype != np.float32:
                    d = d.astype(np.float64)
                d = torch.as_tensor(np.ascontiguousarray(d))
            d = d.to(dev).contiguous()
            if tuple(d.shape) != (self.image_dim[1], self.image_dim[0]):
                raise ValueError(f"depth must be (h={self.image_dim[1]}, w={self.image_dim[0]}), got {tuple(d.shape)}")
            keep.append(d)
            mode = _lib.DEPTH_F32 if d.dtype == torch.float32 else _lib.DEPTH_F64
            dptr = d.data_ptr()
        K = self.intrinsics
        return _lib.FusionView(P=xyz.shape[0], xyz=xyz.data_ptr(), world_to_camera=w2c.data_ptr(),
                               fx=float(K[0][0]), fy=float(K[1][1]), cx=float(K[0][2]), cy=float(K[1][2]),
                               w=int(self.image_dim[0]), h=int(self.image_dim[1]), cut_bound=int(self.cut_bound),
                               vis_thres=float(self.vis_thres), depth_mode=mode, depth=dptr)

    def _ctx(self):
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        return _lib.ctx_for(idx, stream), stream

    def compute_mapping_device(self, world_to_camera, coords, depth=None) -> torch.Tensor:
        """(N,3) int64 CUDA tensor [v, u, mask] — compute_mapping without the host round trip."""
        lib = _lib.load()
        keep: list = []
        with torch.cuda.device(self.device):
            v = self._view(world_to_camera, coords, depth, keep)
            mapping = torch.empty((v.P, 3), dtype=torch.int64, device=self.device)
            ctx, stream = self._ctx()
            _lib.check(lib.sgb_fusion_map(ctx, C.byref(v), mapping.data_ptr(), stream), "sgb_fusion_map")
        return mapping

    def compute_mapping(self, world_to_camera, coords, depth=None, intrinsic=None):
        """Reference signature (fusion_utils.py:30-78): returns (mapping (N,3) int numpy, weight (N,))."""
        mapping = self.compute_mapping_device(world_to_camera, coords, depth).cpu().numpy()
        # `weight` is returned but unused by every caller (fusion_utils.py:76); it depends on the
        # rounded pixel of ALL points, which the device path does not keep, so recompute it here.
        c = np.asarray(coords.detach().cpu() if isinstance(coords, torch.Tensor) else coords, dtype=np.float64)
        w2c = np.asarray(world_to_camera.detach().cpu() if isinstance(world_to_camera, torch.Tensor)
                         else world_to_camera)
        p = np.matmul(w2c.T, np.concatenate([c, np.ones([c.shape[0], 1])], axis=1).T)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = (p[0] * self.intrinsics[0][0]) / p[2] + self.intrinsics[0][2]
            v = (p[1] * self.intrinsics[1][1]) / p[2] + self.intrinsics[1][2]
            pi0, pi1 = np.round(u), np.round(v)
            dist = np.sqrt((pi0 - self.image_dim[0] / 2) ** 2 + (pi1 - self.image_dim[1] / 2) ** 2)
            weight = np.exp(-dist / 10)
        return mapping, weight

    def accumulate(self, world_to_camera, coords, features: torch.Tensor, feat_sum: torch.Tensor,
                   count: torch.Tensor, depth=None) -> torch.Tensor:
        """One fused view of fusion.py:127-144: feat_sum[mask] += features[:, v, u].T ; count[mask] += 1.
        ``features`` is the (C, h, w) fp16/fp32 map of the 2D model; returns a 0-d int32 CUDA tensor
        with the number of Gaussians this view touched."""
        lib = _lib.load()
        dev = self.device
        if features.dtype not in (torch.float16, torch.float32):
            raise TypeError("features must be float16 or float32")
        Cn, h, w = features.shape
        if (w, h) != (self.image_dim[0], self.image_dim[1]):
            raise ValueError("feature map size does not match image_dim")
        feats = features.to(dev).contiguous()
        if feat_sum.dtype != torch.float32 or count.dtype != torch.float32 or not feat_sum.is_contiguous():
            raise TypeError("feat_sum / count must be contiguous float32")
        keep: list = [feats]
        with torch.cuda.device(dev):
            v = self._view(world_to_camera, coords, depth, keep)
            if feat_sum.shape != (v.P, Cn) or count.numel() != v.P:
                raise ValueError("feat_sum must be (P, C) and count (P,) / (P,1)")
            nvis = torch.zeros((), dtype=torch.int32, device=dev)
            ctx, stream = self._ctx()
            dt = _lib.FEAT_F16 if feats.dtype == torch.float16 else _lib.FEAT_F32
            _lib.check(lib.sgb_fusion_accumulate(ctx, C.byref(v), feats.data_ptr(), Cn, dt, feat_sum.data_ptr(),
                                                 count.data_ptr(), nvis.data_ptr(), stream), "sgb_fusion_accumulate")
        return nvis


def normalize_fused(feat_sum: torch.Tensor, count: torch.Tensor) -> None:
    """fusion.py:146-147 in place: count[count == 0] = 1e-5; feat_sum /= count."""
    lib = _lib.load()
    P, Cn = feat_sum.shape
    with torch.cuda.device(feat_sum.device):
        stream = torch.cuda.current_stream(feat_sum.device).cuda_stream
        _lib.check(lib.sgb_fusion_normalize(P, Cn, feat_sum.data_ptr(), count.data_ptr(), stream),
                   "sgb_fusion_normalize")


def fuse_views(gaussians, views, feature_maps, mapper_kwargs: dict, depths=None, every: int = 1):
    """The accumulate loop of fuse_one_scene (fusion.py:57-148) on the device.

    gaussians     object with _xyz, _features_semantic (P,C) f32, _times (P,1) f32 (create_semantic)
    views         sequence with .world_view_transform (4x4, W2C^T) and .intrinsics() / per-view 4x4 K
    feature_maps  sequence (or callable idx -> tensor) of (C,h,w) maps
    depths        None | sequence of depth maps / "surface"
    every         the shipped loop fuses every 5th view (fusion.py:61-62); default here is all."""
    for idx, view in enumerate(views):
        if idx % every != 0:
            continue
        K = view.intrinsics() if callable(getattr(view, "intrinsics", None)) else view.intrinsics
        mapper = PointCloudToImageMapper(intrinsics=K, device=gaussians._xyz.device, **mapper_kwargs)
        fm = feature_maps(idx) if callable(feature_maps) else feature_maps[idx]
        d = None if depths is None else depths[idx]
        mapper.accumulate(view.world_view_transform, gaussians._xyz, fm, gaussians._features_semantic,
                          gaussians._times.view(-1), d)
    normalize_fused(gaussians._features_semantic, gaussians._times.view(-1))
    return gaussians._features_semantic


def fuse_scene(gaussians, views, feature_maps, pipe, background, img_dim, visibility_threshold=0.25,
               cut_boundary=0, depth="render", depth_maps=None, every: int = 5) -> dict:
    """fuse_one_scene (fusion.py:57-148) with every step on the device.

    The reference renders the depth map on the GPU, copies it to the host, projects all Gaussians in numpy,
    gathers the (C,h,w) feature map on the CPU and copies a (P,C) tensor back — per view (fusion.py:106-144).
    Here ``depth="render"`` feeds the rasterizer's median-depth output straight into the fusion kernels.

    depth         "render" (fusion.py:110-120) | "image" (``depth_maps[idx]``, already divided by depth_scale)
                  | "surface" | None
    feature_maps  sequence or callable idx -> (C,h,w) float16/float32 tensor (the 2D model's output)
    every         the shipped loop fuses every 5th view (fusion.py:61-62)
    Returns {"features": (P,C) fused means, "mask": (P,) bool — Gaussians seen by at least one fused view
    (``point_ids`` of fusion.py:148), "views": number of fused views}."""
    from .renderer import render
    if getattr(gaussians, "_features_semantic", None) is None or gaussians._features_semantic.numel() == 0:
        raise ValueError("call gaussians.create_semantic(C) first (fusion.py:52)")
    dev = gaussians._xyz.device
    count = gaussians._times.view(-1)
    fused = 0
    with torch.no_grad():
        for idx, view in enumerate(views):
            if idx % every != 0:
                continue
            K = view.intrinsics() if callable(getattr(view, "intrinsics", None)) else view.intrinsics
            mapper = PointCloudToImageMapper(img_dim, visibility_threshold, cut_boundary, K, device=dev)
            fm = feature_maps(idx) if callable(feature_maps) else feature_maps[idx]
            if depth == "render":
                d = render(view, gaussians, pipe, background, override_shape=img_dim)["depth"][0]
            elif depth == "image":
                d = depth_maps[idx]
            elif depth == "surface":
                d = "surface"
            else:
                d = None
            mapper.accumulate(view.world_view_transform, gaussians._xyz, fm, gaussians._features_semantic, count, d)
            fused += 1
        mask = count > 0
        normalize_fused(gaussians._features_semantic, count)
    return {"features": gaussians._features_semantic, "mask": mask, "views": fused}


# ------------------------------------------------------------------------------------------------------------------
# Fusion by blend weights: the adjoint of rendering (sgb_lift_batch, include/sgb200.h)

def _lift_map(m, idx, Cn, dev, hw):
    """The (C, h, w) map of view idx as the native call reads it; raises on anything it would misread."""
    if not isinstance(m, torch.Tensor):
        raise TypeError(f"feature map {idx} must be a torch.Tensor, got {type(m).__name__}")
    if m.dtype not in (torch.float16, torch.float32):
        raise TypeError(f"feature map {idx} must be float16 or float32, got {m.dtype}")
    if m.device != dev:
        raise ValueError(f"feature map {idx} is on {m.device}, expected {dev}")
    if m.ndim != 3 or m.shape[0] != Cn or m.shape[1] < 1 or m.shape[2] < 1:
        raise ValueError(f"feature map {idx} must be (C={Cn}, h, w), got {tuple(m.shape)}")
    if hw is not None and tuple(m.shape[1:]) != hw:
        raise ValueError(f"feature map {idx} is {tuple(m.shape[1:])}, the other maps of the call are {hw}: the "
                         f"views of one call share the render size")
    return m.contiguous()


def lift_views(gaussians, views, feature_maps, pipe, feat_sum: torch.Tensor, weight_sum: torch.Tensor,
               scaling_modifier: float = 1.0) -> int:
    """Lift 2D feature maps onto the Gaussians by their blend weights, accumulating

        feat_sum[i]  += sum_v sum_p w_i^v(p) F_v[:, p]          weight_sum[i] += sum_v sum_p w_i^v(p)

    where w_i^v(p) = alpha_i T_i is the weight with which the render of view v composites Gaussian i into pixel p (0
    where it is occluded or outside its footprint).  feat_sum is the feature gradient a render_chn backward with the
    map as dL/dout would give, without the colour blend and the rest of the backward; normalize_fused(feat_sum,
    weight_sum) turns it into the weighted mean of the map over the pixels each Gaussian shows in.

    gaussians     GaussianModel-like (get_xyz, get_opacity, get_scaling, get_rotation, get_covariance)
    views         cameras (FoVx, FoVy, world_view_transform, full_proj_transform, camera_center)
    feature_maps  sequence, or callable idx -> map, of (C, h, w) float16 / float32 tensors on the Gaussians' device;
                  views are rendered at the map size (render()'s override_shape), which all maps of a call share
    pipe          compute_cov3d_python, debug and antialiasing are honoured as in render_chn_batch
    feat_sum      (P, C) and weight_sum (P,) or (P, 1): contiguous float32 on the Gaussians' device, added into

    The views go to the native call in batches of at most 8 consecutive views whose maps share a dtype.  A sequence
    of maps is checked in full before the first native call, a callable's maps batch by batch as they are fetched:
    TypeError for a non-tensor or a dtype other than float16 / float32, ValueError for a wrong shape or device or a
    map size that differs from the call's first map.  Returns the number of views lifted."""
    from . import channel_rasterization as chn
    from .rasterizer import _cameras, _make_inputs, _ptrs, _stream_ctx
    from .renderer import _antialiasing, _prepare
    views = list(views)
    xyz = gaussians.get_xyz
    dev, P = xyz.device, xyz.shape[0]
    for name, t, shape in (("feat_sum", feat_sum, None), ("weight_sum", weight_sum, (P,))):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
            raise TypeError(f"{name} must be a float32 tensor")
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, expected {dev}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous (it is accumulated in place)")
    if feat_sum.ndim != 2 or feat_sum.shape[0] != P:
        raise ValueError(f"feat_sum must be (P={P}, C), got {tuple(feat_sum.shape)}")
    if weight_sum.numel() != P:
        raise ValueError(f"weight_sum must hold P={P} entries, got {tuple(weight_sum.shape)}")
    Cn = feat_sum.shape[1]
    fetch = feature_maps if callable(feature_maps) else feature_maps.__getitem__
    hw = None
    if not callable(feature_maps):
        if len(feature_maps) < len(views):
            raise ValueError(f"{len(views)} views but {len(feature_maps)} feature maps")
        for i in range(len(views)):
            hw = tuple(_lift_map(feature_maps[i], i, Cn, dev, hw).shape[1:])
    if not xyz.is_cuda:
        raise ValueError(f"the Gaussians are on {dev}: lifting runs on a CUDA device only (there is no CPU path)")
    if not views:
        return 0
    lib = _lib.load()
    debug = bool(getattr(pipe, "debug", False))
    with torch.no_grad(), torch.cuda.device(dev):
        i = 0
        bg = carry = None   # carry: a fetched map of the other dtype, the first of the next batch
        while i < len(views):
            maps = [carry if carry is not None else _lift_map(fetch(i), i, Cn, dev, hw)]
            carry = None
            hw = tuple(maps[0].shape[1:])
            while i + len(maps) < len(views) and len(maps) < _lib.MAX_BATCH:
                m = _lift_map(fetch(i + len(maps)), i + len(maps), Cn, dev, hw)
                if m.dtype != maps[0].dtype:
                    carry = m
                    break
                maps.append(m)
            h, w = hw
            batch = views[i:i + len(maps)]
            if bg is None:
                # the Gaussian-side tensors once per call, as render_chn_batch prepares them; any override colour
                # keeps _prepare from evaluating SH colours, which a lift does not read
                _, common0, call = _prepare(batch[0], gaussians, pipe, scaling_modifier, override_color=feat_sum,
                                            override_shape=(w, h), foreground=None, world_rotate=None)
                bg = torch.zeros(Cn, device=dev)   # _make_inputs wants a background; the native call takes none
            settings = [chn.GaussianRasterizationSettings(
                bg=bg, debug=debug, num_channels=Cn,
                **dict(common0, tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
                       viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
                       campos=cam.camera_center)) for cam in batch]
            inp, cameras, keep, _ = _make_inputs(_cameras(settings), bg, call["means3D"], None,
                                                 call["opacities"], call["scales"], call["rotations"], scaling_modifier,
                                                 call["cov3D_precomp"], h, w, None, 0, False, debug, Cn,
                                                 antialiasing=_antialiasing(pipe))
            inp.background = None
            stream, ctx = _stream_ctx(dev)
            dt = _lib.FEAT_F16 if maps[0].dtype == torch.float16 else _lib.FEAT_F32
            _lib.check(lib.sgb_lift_batch(ctx, C.byref(inp), len(maps), cameras, _ptrs(maps), dt,
                                          feat_sum.data_ptr(), weight_sum.data_ptr(), stream), "sgb_lift_batch")
            i += len(maps)
    return len(views)


def lift_scene(gaussians, views, feature_maps, pipe, every: int = 5) -> dict:
    """The counterpart of fuse_scene that needs no depth map, visibility threshold or boundary cut: every view
    ``idx % every == 0`` is lifted with lift_views (occlusion comes from the render's transmittance), and each
    Gaussian gets the weighted mean of the feature-map pixels it shows in.

    Writes the means into ``gaussians._features_semantic`` (create_semantic(C) first) and the weight sums into
    ``gaussians._times``.  Returns {"features": (P, C) float32, "mask": (P,) bool, weight sum > 0 (a Gaussian no
    lifted pixel shows has features 0), "views": number of lifted views, "weights": (P,) float32 weight sums}, which
    io_formats.save_fused_features and the evaluation code take as they take fuse_scene's result."""
    if getattr(gaussians, "_features_semantic", None) is None or gaussians._features_semantic.numel() == 0:
        raise ValueError("call gaussians.create_semantic(C) first")
    views = list(views)
    sel = list(range(0, len(views), every))
    maps = (lambda k: feature_maps(sel[k])) if callable(feature_maps) else [feature_maps[i] for i in sel]
    feats, weights = gaussians._features_semantic, gaussians._times.view(-1)
    with torch.no_grad():
        feats.zero_()
        weights.zero_()
        n = lift_views(gaussians, [views[i] for i in sel], maps, pipe, feats, weights)
        mask = weights > 0
        normalize_fused(feats, weights.clone())   # the normaliser marks zero sums 1e-5; the weights stay as summed
    return {"features": feats, "mask": mask, "views": n, "weights": weights}
