"""The single-view C entry points sgb_forward_geometry / sgb_forward_render / sgb_backward, called directly through
ctypes the way a C++ caller uses them (INTEGRATION.md).  The Python layer renders one view through the batched entry
points with V = 1, so these calls are checked here against it: the forward bit for bit, the gradients to the float
atomics' tolerance."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from util import dev_cam, dev_scene, frac_bad  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.rasterizer import _C_chn, _C_rgbd  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu

GRADS = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
         "dL_drotations")   # the order of rasterize_gaussians_backward's return tuple


@pytest.mark.parametrize("Cn,use_features", [(3, False),     # SH path, RGB + depth
                                             (64, True)])    # precomputed features
def test_single_view_entry_points_match_python_path(Cn, use_features):
    dev = torch.device("cuda:0")
    P, W, H = 20000, 320, 240
    scene = make_scene(P, seed=11, sh=not use_features, channels=Cn if use_features else 0)
    sc, cm = dev_scene(scene, dev), dev_cam(orbit_cameras(4, W, H)[1], dev)
    bg = torch.linspace(0.0, 0.5, Cn, device=dev)
    empty = torch.Tensor([])
    colors = sc["features"] if use_features else empty
    sh, degree = (empty, 0) if use_features else (sc["shs"], 3)
    M = 0 if use_features else sh.shape[1]
    dL = torch.as_tensor(np.random.default_rng(4).standard_normal((Cn, H, W)).astype(np.float32), device=dev)

    cam = [cm["viewmatrix"], cm["projmatrix"], cm["tanfovx"], cm["tanfovy"]]
    fwd = [bg, sc["means3D"], colors, sc["opacities"], sc["scales"], sc["rotations"], 1.0, empty, *cam, H, W, sh,
           degree, cm["campos"], False]
    if use_features:
        R, color, radii, geom, binning, img = _C_chn.rasterize_gaussians(*fwd, False, Cn)
        depth = None
        bwd = _C_chn.rasterize_gaussians_backward
    else:
        R, color, radii, geom, binning, img, depth = _C_rgbd.rasterize_gaussians(*fwd)
        bwd = _C_rgbd.rasterize_gaussians_backward
    want = dict(zip(GRADS, bwd(bg, sc["means3D"], radii, colors, sc["scales"], sc["rotations"], 1.0, empty, *cam, dL,
                               sh, degree, cm["campos"], geom, R, binning, img, *([False] if use_features else []))))

    lib = _lib.load()
    ptr = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()
    inp = _lib.ViewInputs(
        P=P, D=degree, M=M, W=W, H=H, C=Cn, background=ptr(bg), means3D=ptr(sc["means3D"]), shs=ptr(sh),
        colors_precomp=ptr(colors), opacities=ptr(sc["opacities"]), scales=ptr(sc["scales"]), scale_modifier=1.0,
        rotations=ptr(sc["rotations"]), cov3D_precomp=None, viewmatrix=ptr(cm["viewmatrix"]),
        projmatrix=ptr(cm["projmatrix"]), campos=ptr(cm["campos"]), tan_fovx=cm["tanfovx"], tan_fovy=cm["tanfovy"],
        prefiltered=0, debug=0)
    u8 = dict(dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ctx = C.c_void_p()
    _lib.check(lib.sgb_ctx_create(C.byref(ctx), dev.index), "sgb_ctx_create")
    try:
        radii2 = torch.empty((P,), dtype=torch.int32, device=dev)
        geom2 = torch.empty((lib.sgb_geometry_bytes(P),), **u8)
        img2 = torch.empty((lib.sgb_image_bytes(W, H),), **u8)
        R2 = C.c_int64(0)
        _lib.check(lib.sgb_forward_geometry(ctx, C.byref(inp), geom2.data_ptr(), radii2.data_ptr(), C.byref(R2),
                                            stream), "sgb_forward_geometry")
        binning2 = torch.empty((lib.sgb_binning_bytes(R2.value),), **u8)
        color2 = torch.empty((Cn, H, W), device=dev)
        depth2 = None if use_features else torch.empty((1, H, W), device=dev)
        _lib.check(lib.sgb_forward_render(ctx, C.byref(inp), R2.value, geom2.data_ptr(), binning2.data_ptr(),
                                          img2.data_ptr(), radii2.data_ptr(), color2.data_ptr(), ptr(depth2), stream),
                   "sgb_forward_render")
        got = {k: torch.zeros_like(want[k]) for k in GRADS}
        conic = torch.zeros((P, 2, 2), device=dev)
        grads = _lib.ViewGrads(dL_dconic=conic.data_ptr(), **{k: ptr(t) for k, t in got.items()})
        _lib.check(lib.sgb_backward(ctx, C.byref(inp), R2.value, radii2.data_ptr(), geom2.data_ptr(),
                                    binning2.data_ptr(), img2.data_ptr(), dL.data_ptr(), C.byref(grads), stream),
                   "sgb_backward")
    finally:
        torch.cuda.synchronize(dev)
        lib.sgb_ctx_destroy(ctx)

    assert R > 0 and R2.value == R
    assert torch.equal(radii2, radii)
    assert torch.equal(color2.view(torch.int32), color.view(torch.int32))
    if depth is not None:
        assert torch.equal(depth2.view(torch.int32), depth.view(torch.int32))
    for name in GRADS:
        if want[name].numel() == 0:   # dL_dsh without SH
            continue
        assert float(want[name].abs().max()) > 0, name
        # both sides sum fp32 partial gradients with red.global in scheduling order
        assert frac_bad(got[name], want[name], rtol=1e-4, atol_scale=1e-4) == 0.0, name
