"""Shared helpers of the test-suite: run the product (through its public Python API / C-ABI),
the compiled reference (oracle/_ref) and the CPU oracle on the same seeded scene."""
from __future__ import annotations

import hashlib
import math
import os
import zlib

import numpy as np
import torch

from semantic_gaussians_b200.scene_synth import SynthCamera, SynthScene


def dev_scene(scene: SynthScene, dev, requires_grad=False):
    t = lambda a: None if a is None else torch.as_tensor(a, device=dev).contiguous().requires_grad_(requires_grad)
    return dict(means3D=t(scene.xyz), scales=t(scene.scales), rotations=t(scene.rotations),
                opacities=t(scene.opacity), shs=t(scene.shs), features=t(scene.features))


def dev_cam(cam: SynthCamera, dev):
    t = lambda a: torch.as_tensor(a, device=dev).contiguous()
    return dict(viewmatrix=t(cam.world_view_transform), projmatrix=t(cam.full_proj_transform),
                campos=t(cam.camera_center), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
                W=cam.image_width, H=cam.image_height)


def run_ours(variant, sc, cm, bg, *, use_features, sh_degree=3, debug=False, cov3D_precomp=None, scale_modifier=1.0):
    """Forward through the drop-in modules; returns dict with outputs and the autograd handles."""
    if variant == "rgbd":
        from semantic_gaussians_b200 import rgbd_rasterization as mod
        rs = mod.GaussianRasterizationSettings(
            image_height=cm["H"], image_width=cm["W"], tanfovx=cm["tanfovx"], tanfovy=cm["tanfovy"], bg=bg,
            scale_modifier=scale_modifier, viewmatrix=cm["viewmatrix"], projmatrix=cm["projmatrix"],
            sh_degree=sh_degree, campos=cm["campos"], prefiltered=False, debug=debug)
    else:
        from semantic_gaussians_b200 import channel_rasterization as mod
        C = sc["features"].shape[1] if use_features else 3
        rs = mod.GaussianRasterizationSettings(
            image_height=cm["H"], image_width=cm["W"], tanfovx=cm["tanfovx"], tanfovy=cm["tanfovy"], bg=bg,
            scale_modifier=scale_modifier, viewmatrix=cm["viewmatrix"], projmatrix=cm["projmatrix"],
            sh_degree=sh_degree, campos=cm["campos"], prefiltered=False, debug=debug, num_channels=C)
    rast = mod.GaussianRasterizer(rs)
    means2D = torch.zeros_like(sc["means3D"], requires_grad=sc["means3D"].requires_grad)
    kw = dict(means3D=sc["means3D"], means2D=means2D, opacities=sc["opacities"])
    if use_features:
        kw["colors_precomp"] = sc["features"]
    else:
        kw["shs"] = sc["shs"]
    if cov3D_precomp is not None:
        kw["cov3D_precomp"] = cov3D_precomp
    else:
        kw["scales"], kw["rotations"] = sc["scales"], sc["rotations"]
    out = rast(**kw)
    res = dict(color=out[0], radii=out[1], means2D=means2D)
    if variant == "rgbd":
        res["depth"] = out[2]
    return res


def ours_state(sc, cm, C, *, use_features, want_depth=False, sh_degree=3):
    """Forward through the pybind-like _C surface, plus every opaque state field as tensors."""
    import ctypes as Ct

    from semantic_gaussians_b200 import _lib
    from semantic_gaussians_b200.rasterizer import _C_chn, _C_rgbd
    dev = sc["means3D"].device
    empty = torch.Tensor([])
    bg = torch.zeros(C, device=dev)
    colors = sc["features"] if use_features else empty
    sh = empty if use_features else sc["shs"]
    args = [bg, sc["means3D"], colors, sc["opacities"], sc["scales"], sc["rotations"], 1.0, empty, cm["viewmatrix"],
            cm["projmatrix"], cm["tanfovx"], cm["tanfovy"], cm["H"], cm["W"], sh, sh_degree, cm["campos"], False]
    if want_depth:
        R, color, radii, geom, binning, img, depth = _C_rgbd.rasterize_gaussians(*args)
    else:
        R, color, radii, geom, binning, img = _C_chn.rasterize_gaussians(*args, False, C)
        depth = None
    lib = _lib.load()
    P, W, H = sc["means3D"].shape[0], cm["W"], cm["H"]
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    spec = dict(depths=(torch.float32, (P,)), means2D=(torch.float32, (P, 2)), conic_opacity=(torch.float32, (P, 4)),
                cov3D=(torch.float32, (P, 6)), rgb=(torch.float32, (P, 3)), clamped=(torch.uint8, (P, 3)),
                tiles_touched=(torch.int32, (P,)), point_list=(torch.int32, (max(R, 1),)),
                ranges=(torch.int32, (tiles, 2)), n_contrib=(torch.int32, (H * W,)), final_T=(torch.float32, (H * W,)))
    st = {}
    stream = torch.cuda.current_stream(dev).cuda_stream
    for name, (dt, shape) in spec.items():
        t = torch.zeros(shape, dtype=dt, device=dev)
        n = lib.sgb_state_field(name.encode(), P, R, W, H, geom.data_ptr(), binning.data_ptr(), img.data_ptr(),
                                t.data_ptr(), stream)
        assert n >= 0, lib.sgb_last_error()
        st[name] = t[:R] if name == "point_list" else t
    torch.cuda.synchronize(dev)
    st.update(R=R, color=color, radii=radii, depth=depth)
    return st


GOLDEN_REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")


def _np(t):
    return t.detach().contiguous().cpu().numpy() if isinstance(t, torch.Tensor) else np.ascontiguousarray(t)


class RefRecord:
    """What one test compares against the compiled reference rasterizer (oracle/_ref), stored in
    tests/golden/ref/<case>.npz so that the comparison runs where the reference is not built: arrays compared bit
    for bit as the SHA-256 of their bytes, arrays compared to a tolerance as a fixed seeded sample of their entries
    plus the whole array's max |x|.  With SGB_RECORD_REF=1 the test runs the reference live, checks against the full
    arrays and rewrites the record (`SGB_RECORD_REF=1 python -m pytest tests -m gpu` with oracle/_ref built).  `ref`
    arguments are callables that produce the live reference array; they are only called when recording."""
    SAMPLE = 16384   # 64 KB per array: a record of seven sampled arrays stays well under 1 MB

    def __init__(self, case):
        self.path = os.path.join(GOLDEN_REF, case + ".npz")
        self.live = os.environ.get("SGB_RECORD_REF") == "1"
        self.data = {} if self.live else dict(np.load(self.path))

    def save(self):
        if self.live:
            os.makedirs(GOLDEN_REF, exist_ok=True)
            np.savez_compressed(self.path, **self.data)

    @staticmethod
    def _digest(a):
        a = _np(a)
        h = hashlib.sha256(str((a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
        return np.frombuffer(h.digest(), np.uint8)

    def equal(self, key, ours, ref=None):
        """Same dtype, shape and bytes as the reference array."""
        if self.live:
            self.data[key + ".sha256"] = self._digest(ref())
        return bool(np.array_equal(self._digest(ours), self.data[key + ".sha256"]))

    def _pair(self, key, ours, ref):
        a = _np(ours).astype(np.float64).reshape(-1)
        if self.live:
            b = _np(ref()).astype(np.float64).reshape(-1)
            assert a.size == b.size, key
            idx = self._index(key, b.size)
            self.data[key + ".sample"] = b[idx].astype(np.float32)   # the reference computes in fp32
            self.data[key + ".maxabs"] = np.float64(np.abs(b).max() if b.size else 0.0)
            self.data[key + ".size"] = np.int64(b.size)
            return a, b, float(self.data[key + ".maxabs"])
        assert a.size == int(self.data[key + ".size"]), key
        return a[self._index(key, a.size)], self.data[key + ".sample"].astype(np.float64), float(self.data[key + ".maxabs"])

    def _index(self, key, n):
        if n <= self.SAMPLE:
            return np.arange(n)
        rng = np.random.default_rng(zlib.crc32(key.encode()))
        return np.unique(rng.integers(0, n, self.SAMPLE))

    def frac_bad(self, key, ours, ref=None, rtol=1e-4, atol_scale=1e-4):
        """frac_bad() against the reference: over the whole array when recording, over the sample otherwise."""
        a, b, m = self._pair(key, ours, ref)
        return float((np.abs(a - b) > rtol * np.abs(b) + atol_scale * m).mean()) if b.size else 0.0

    def max_abs_diff(self, key, ours, ref=None):
        """(max |ours - ref|, max |ref|), the first over the whole array when recording, over the sample otherwise."""
        a, b, m = self._pair(key, ours, ref)
        return (float(np.abs(a - b).max()) if b.size else 0.0), m

    def rel_err(self, key, ours, ref=None):
        d, m = self.max_abs_diff(key, ours, ref)
        return d / (m + 1e-30)


def rel_err(a, b):
    """max |a-b| / max|b| over the tensor (b = reference)."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b)).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def frac_bad(a, b, rtol=1e-4, atol_scale=1e-4):
    """Fraction of entries with |a-b| > rtol*|b| + atol_scale*max|b|."""
    a = a.detach().double().cpu().reshape(-1)
    b = (b.detach().double().cpu() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b)).double()).reshape(-1)
    tol = rtol * b.abs() + atol_scale * b.abs().max()
    return float(((a - b).abs() > tol).double().mean())
