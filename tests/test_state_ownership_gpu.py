"""Render and backward read only the caller's states, radii and instance count (include/sgb200.h): calls for
different views may interleave on one ctx, a batched render may take any subset or order of a geometry batch's
views, a render may run on another ctx than its geometry call, and a lift in between changes nothing.  Every case is
compared with the plain geometry -> render -> backward sequence of the same view on a fresh ctx: the forward bit for
bit, the gradients to the float atomics' tolerance."""
import contextlib
import ctypes as Ct
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from raster_check import read_state  # noqa: E402
from util import dev_cam, dev_scene, frac_bad  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
P, W, H = 20000, 320, 240
BITWISE = ("color", "depth", "radii", "point_list", "ranges", "n_contrib", "final_T")
GRADS = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_dmeans3D", "dL_dcov3D", "dL_dsh",
         "dL_dscales", "dL_drotations")
CONFIGS = pytest.mark.parametrize("Cn,use_features", [(3, False),    # SH colours, RGB + depth
                                                      (64, True)])   # colors_precomp, weight-pool path


class Rig:
    """One seeded scene, four orbit cameras and a fixed dL/dout per camera, driven through the batched C ABI.  A view
    is a dict: its camera index, then the states and outputs each call fills in."""

    def __init__(self, Cn, use_features):
        self.lib = _lib.load()
        self.Cn, self.use_sh = Cn, not use_features
        scene = make_scene(P, seed=11, sh=self.use_sh, channels=0 if self.use_sh else Cn)
        self.sc = dev_scene(scene, DEV)
        self.cams = [dev_cam(c, DEV) for c in orbit_cameras(4, W, H)]
        self.bg = torch.linspace(0.0, 0.5, Cn, device=DEV)
        self.M = self.sc["shs"].shape[1] if self.use_sh else 0
        self.inp = self.inputs(C=Cn, D=3 if self.use_sh else 0, M=self.M, background=self.bg.data_ptr(),
                               shs=self.sc["shs"].data_ptr() if self.use_sh else None,
                               colors_precomp=None if self.use_sh else self.sc["features"].data_ptr())
        g = torch.Generator(device=DEV).manual_seed(4)
        self.dL = [torch.randn((Cn, H, W), device=DEV, generator=g) for _ in self.cams]
        self.stream = torch.cuda.current_stream(DEV).cuda_stream

    def inputs(self, **kw):
        """sgb_view_inputs of the scene; the camera fields are taken from the sgb_camera array of each call."""
        base = dict(P=P, W=W, H=H, means3D=self.sc["means3D"].data_ptr(), opacities=self.sc["opacities"].data_ptr(),
                    scales=self.sc["scales"].data_ptr(), scale_modifier=1.0, rotations=self.sc["rotations"].data_ptr(),
                    cov3D_precomp=None, viewmatrix=None, projmatrix=None, campos=None, tan_fovx=0.0, tan_fovy=0.0,
                    prefiltered=0, debug=0)
        base.update(kw)
        return _lib.ViewInputs(**base)

    def camera_array(self, idx):
        cms = [self.cams[i] for i in idx]
        return (_lib.Camera * len(idx))(*[_lib.Camera(c["viewmatrix"].data_ptr(), c["projmatrix"].data_ptr(),
                                                      c["campos"].data_ptr(), c["tanfovx"], c["tanfovy"]) for c in cms])

    @contextlib.contextmanager
    def ctx(self):
        ctx = Ct.c_void_p()
        _lib.check(self.lib.sgb_ctx_create(Ct.byref(ctx), DEV.index), "sgb_ctx_create")
        try:
            yield ctx
        finally:
            torch.cuda.synchronize(DEV)
            self.lib.sgb_ctx_destroy(ctx)

    @staticmethod
    def _ptrs(views, key):
        return (Ct.c_void_p * len(views))(*[v[key].data_ptr() for v in views])

    def geometry(self, ctx, idx):
        """sgb_forward_geometry_batch of cameras idx; one view dict per camera."""
        u8 = dict(dtype=torch.uint8, device=DEV)
        views = [dict(cam=i, radii=torch.empty((P,), dtype=torch.int32, device=DEV),
                      geom=torch.empty((self.lib.sgb_geometry_bytes(P),), **u8)) for i in idx]
        Rs = (Ct.c_int64 * len(idx))()
        _lib.check(self.lib.sgb_forward_geometry_batch(ctx, Ct.byref(self.inp), len(idx), self.camera_array(idx),
                                                       self._ptrs(views, "geom"), self._ptrs(views, "radii"), Rs,
                                                       self.stream), "sgb_forward_geometry_batch")
        for v, R in zip(views, Rs):
            v["R"] = R
        return views

    def render(self, ctx, views):
        """sgb_forward_render_batch of geometry views, into fresh binning / image states and outputs: new view dicts
        (a geometry view can be rendered more than once)."""
        u8 = dict(dtype=torch.uint8, device=DEV)
        out = [dict(v, binning=torch.empty((self.lib.sgb_binning_bytes(v["R"]),), **u8),
                    img=torch.empty((self.lib.sgb_image_bytes(W, H),), **u8),
                    color=torch.empty((self.Cn, H, W), device=DEV),
                    depth=torch.empty((1, H, W), device=DEV) if self.use_sh else None) for v in views]
        V = len(out)
        Rs = (Ct.c_int64 * V)(*[v["R"] for v in out])
        _lib.check(self.lib.sgb_forward_render_batch(ctx, Ct.byref(self.inp), V, self.camera_array([v["cam"] for v in out]),
                                                     Rs, self._ptrs(out, "geom"), self._ptrs(out, "binning"),
                                                     self._ptrs(out, "img"), self._ptrs(out, "radii"),
                                                     self._ptrs(out, "color"),
                                                     self._ptrs(out, "depth") if self.use_sh else None, self.stream),
                   "sgb_forward_render_batch")
        return out

    def backward(self, ctx, views):
        """sgb_backward_batch of rendered views with their camera's dL/dout; each view gets its own gradients."""
        z = lambda *s: torch.zeros(s, device=DEV)
        for v in views:
            v["grads"] = dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 4), dL_dopacity=z(P), dL_dcolors=z(P, self.Cn),
                              dL_dmeans3D=z(P, 3), dL_dcov3D=z(P, 6), dL_dsh=z(P, self.M, 3) if self.use_sh else None,
                              dL_dscales=z(P, 3), dL_drotations=z(P, 4))
        V = len(views)
        gr = (_lib.ViewGrads * V)(*[_lib.ViewGrads(**{k: None if t is None else t.data_ptr()
                                                      for k, t in v["grads"].items()}) for v in views])
        Rs = (Ct.c_int64 * V)(*[v["R"] for v in views])
        dL = (Ct.c_void_p * V)(*[self.dL[v["cam"]].data_ptr() for v in views])
        _lib.check(self.lib.sgb_backward_batch(ctx, Ct.byref(self.inp), V, self.camera_array([v["cam"] for v in views]),
                                               Rs, self._ptrs(views, "radii"), self._ptrs(views, "geom"),
                                               self._ptrs(views, "binning"), self._ptrs(views, "img"), dL, gr,
                                               self.stream), "sgb_backward_batch")
        return views

    def result(self, v):
        """The forward outputs and states of a rendered view, plus its gradients when it has them."""
        st = read_state(self.lib, P, v["R"], W, H, v["geom"], v["binning"], v["img"])
        res = {k: st[k] for k in ("point_list", "ranges", "n_contrib", "final_T")}
        res.update(R=v["R"], color=v["color"], depth=v["depth"], radii=v["radii"], grads=v.get("grads"))
        return res

    def plain(self, i, backward=True):
        """Camera i alone on a fresh ctx: geometry, render and (optionally) backward."""
        with self.ctx() as ctx:
            v = self.render(ctx, self.geometry(ctx, [i]))
            if backward:
                self.backward(ctx, v)
        return self.result(v[0])


def assert_same(got, want):
    assert got["R"] == want["R"] > 0
    for k in BITWISE:
        if want[k] is None:
            continue
        a, b = got[k].contiguous(), want[k].contiguous()
        assert a.shape == b.shape and torch.equal(a.view(torch.uint8), b.view(torch.uint8)), k
    if want["grads"] is None:
        return
    for k in GRADS:
        w = want["grads"][k]
        if w is None:
            continue
        # both sides sum fp32 partial gradients with red.global in scheduling order
        assert frac_bad(got["grads"][k], w, rtol=1e-4, atol_scale=1e-4) == 0.0, k
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dcolors", "dL_dmeans3D"):
        assert float(want["grads"][k].abs().max()) > 0, k


@CONFIGS
def test_interleaved_single_views(Cn, use_features):
    """geometry(A), geometry(B), render(B), render(A), backward(A), backward(B) on one ctx."""
    rig = Rig(Cn, use_features)
    A, B = 0, 1
    with rig.ctx() as ctx:
        ga, = rig.geometry(ctx, [A])
        gb, = rig.geometry(ctx, [B])
        rb, = rig.render(ctx, [gb])
        ra, = rig.render(ctx, [ga])
        rig.backward(ctx, [ra])
        rig.backward(ctx, [rb])
    assert ra["R"] != rb["R"]
    assert_same(rig.result(ra), rig.plain(A))
    assert_same(rig.result(rb), rig.plain(B))


@CONFIGS
def test_batch_render_of_any_subset_and_order(Cn, use_features):
    """One geometry batch of 4 views, rendered as [2, 0, 3, 1] and as [3, 1]: every view equals its V = 1 render."""
    rig = Rig(Cn, use_features)
    with rig.ctx() as ctx:
        geo = rig.geometry(ctx, [0, 1, 2, 3])
        permuted = rig.render(ctx, [geo[i] for i in (2, 0, 3, 1)])
        subset = rig.render(ctx, [geo[i] for i in (3, 1)])
    want = {i: rig.plain(i, backward=False) for i in range(4)}
    for v in permuted + subset:
        assert_same(rig.result(v), want[v["cam"]])


@CONFIGS
def test_render_on_another_ctx_and_after_a_lift(Cn, use_features):
    """Geometry on one ctx, render and backward on another; and geometry(A), a lift of another camera with the same P
    on the same ctx, then render and backward of A."""
    rig = Rig(Cn, use_features)
    A, B = 2, 3
    want = rig.plain(A)
    with rig.ctx() as ctx1, rig.ctx() as ctx2:
        ga = rig.geometry(ctx1, [A])
        ra = rig.backward(ctx2, rig.render(ctx2, ga))
    assert_same(rig.result(ra[0]), want)

    Cl = 16
    lift_inp = rig.inputs(C=Cl, D=0, M=0, background=None, shs=None, colors_precomp=None)
    fmap = torch.randn((Cl, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    feat_sum, weight_sum = torch.zeros((P, Cl), device=DEV), torch.zeros(P, device=DEV)
    with rig.ctx() as ctx:
        ga = rig.geometry(ctx, [A])
        _lib.check(rig.lib.sgb_lift_batch(ctx, Ct.byref(lift_inp), 1, rig.camera_array([B]),
                                          (Ct.c_void_p * 1)(fmap.data_ptr()), _lib.FEAT_F32, feat_sum.data_ptr(),
                                          weight_sum.data_ptr(), rig.stream), "sgb_lift_batch")
        ra = rig.backward(ctx, rig.render(ctx, ga))
    assert float(weight_sum.max()) > 0
    assert_same(rig.result(ra[0]), want)


def test_geometry_scratch_does_not_grow_with_the_batch():
    """The depth order and the scan live in the caller's geometry states: the ctx's geometry scratch is one slice
    whatever the number of views."""
    rig = Rig(3, False)
    scratch = {}
    for V in (1, 8):
        with rig.ctx() as ctx:
            rig.geometry(ctx, [i % 4 for i in range(V)])
            torch.cuda.synchronize(DEV)
            scratch[V] = rig.lib.sgb_ctx_scratch_bytes(ctx)
    assert 0 < scratch[8] < 1.5 * scratch[1], scratch
