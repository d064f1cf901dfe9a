"""The weight pool of the C > 4 blend (the per-tile alpha * T rows that the forward builds and the backward reuses):
a backward whose views lost their pool slots rebuilds them, and a first forward on a fresh ctx that overflows the
first guess of the pool size grows the pool and repeats its alpha pass, with results identical to a warm ctx."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blend_ref as br  # noqa: E402
from test_batch_gpu import Pipe, _cams, _grads, _model  # noqa: E402
from raster_check import FRAGILE_MAX, read_state  # noqa: E402
from util import dev_cam, dev_scene, frac_bad  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.renderer import render_chn, render_chn_batch  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu


def test_batch_backward_rebuilds_recycled_slots():
    """A full batch, then forwards of other views on the same ctx that take over the least recently used slots (the
    batch's first views), then the batch's backward: those views' rows are rebuilt under one stream sync."""
    dev = torch.device("cuda:0")
    C_, W, H, V, extra = 64, 320, 240, _lib.MAX_BATCH, 3
    pc, feats, leaves = _model(30000, C_, dev, seed=13)
    cams = _cams(V + extra, W, H, dev)
    bg = torch.linspace(0.0, 0.2, C_, device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    dLs = [torch.randn((C_, H, W), device=dev, generator=g) for _ in range(V)]

    for c, d in zip(cams[:V], dLs):   # reference: strictly interleaved forward / backward per view
        render_chn(c, pc, Pipe, bg, num_channels=C_, override_color=feats)["render"].backward(d)
    want = _grads(leaves, feats)

    batch = render_chn_batch(cams[:V], pc, Pipe, bg, num_channels=C_, override_color=feats)
    # kept alive until the end, so that each of these forwards holds its own binning state and thereby its own slot
    others = [render_chn(c, pc, Pipe, bg, num_channels=C_, override_color=feats) for c in cams[V:]]
    sum((o["render"] * d).sum() for o, d in zip(batch, dLs)).backward()
    got = _grads(leaves, feats)
    for a, b in zip(want, got):
        assert frac_bad(b, a, rtol=1e-4, atol_scale=1e-4) == 0.0
    del others


def test_first_forward_on_fresh_ctx_overflows_and_retries():
    """A dense, faint scene needs far more than the first guess of 8 chunks (128 entries) per tile, so the first alpha
    pass on a fresh ctx overflows the pool and runs again into a larger one."""
    dev = torch.device("cuda:0")
    P, W, H, Cn = 100000, 128, 96, 16
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    scene = make_scene(P, seed=21, channels=Cn, scale_mean=0.05)
    scene.opacity[:] = 0.02
    sc, cm = dev_scene(scene, dev), dev_cam(orbit_cameras(2, W, H)[0], dev)
    bg = torch.linspace(0.0, 0.5, Cn, device=dev)
    ptr = lambda t: None if t is None else t.data_ptr()
    inp = _lib.ViewInputs(
        P=P, D=0, M=0, W=W, H=H, C=Cn, background=ptr(bg), means3D=ptr(sc["means3D"]), shs=None,
        colors_precomp=ptr(sc["features"]), opacities=ptr(sc["opacities"]), scales=ptr(sc["scales"]),
        scale_modifier=1.0, rotations=ptr(sc["rotations"]), cov3D_precomp=None, viewmatrix=ptr(cm["viewmatrix"]),
        projmatrix=ptr(cm["projmatrix"]), campos=ptr(cm["campos"]), tan_fovx=cm["tanfovx"], tan_fovy=cm["tanfovy"],
        prefiltered=0, debug=0)
    lib = _lib.load()
    u8 = dict(dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ctx = C.c_void_p()
    _lib.check(lib.sgb_ctx_create(C.byref(ctx), dev.index), "sgb_ctx_create")

    def forward():
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        geom = torch.empty((lib.sgb_geometry_bytes(P),), **u8)
        img = torch.empty((lib.sgb_image_bytes(W, H),), **u8)
        R = C.c_int64(0)
        _lib.check(lib.sgb_forward_geometry(ctx, C.byref(inp), geom.data_ptr(), radii.data_ptr(), C.byref(R), stream),
                   "sgb_forward_geometry")
        binning = torch.empty((lib.sgb_binning_bytes(R.value),), **u8)
        color = torch.empty((Cn, H, W), device=dev)
        _lib.check(lib.sgb_forward_render(ctx, C.byref(inp), R.value, geom.data_ptr(), binning.data_ptr(),
                                          img.data_ptr(), radii.data_ptr(), color.data_ptr(), None, stream),
                   "sgb_forward_render")
        return R.value, radii, geom, binning, img, color

    try:
        R, radii, geom, binning, img, color = forward()
        chunks = lib.sgb_ctx_view_stat(ctx, 1)
        R2, radii2, _, _, _, color2 = forward()
        st = read_state(lib, P, R, W, H, geom, binning, img)
        args = (st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], sc["features"], bg, W, H)
        want = br.blend_forward(*args)
        dL = torch.as_tensor(np.random.default_rng(6).standard_normal((Cn, H * W)).astype(np.float32), device=dev)
        dL[:, want["fragile"]] = 0.0   # no gradient from pixels whose blend fp32 rounding could decide otherwise
        dL = dL.reshape(Cn, H, W)
        grads = {k: torch.zeros(s, device=dev) for k, s in (
            ("dL_dmeans2D", (P, 3)), ("dL_dconic", (P, 2, 2)), ("dL_dopacity", (P, 1)), ("dL_dcolors", (P, Cn)),
            ("dL_dmeans3D", (P, 3)), ("dL_dcov3D", (P, 6)), ("dL_dscales", (P, 3)), ("dL_drotations", (P, 4)))}
        gr = _lib.ViewGrads(**{k: t.data_ptr() for k, t in grads.items()})
        _lib.check(lib.sgb_backward(ctx, C.byref(inp), R, radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
                                    img.data_ptr(), dL.data_ptr(), C.byref(gr), stream), "sgb_backward")
    finally:
        torch.cuda.synchronize(dev)
        lib.sgb_ctx_destroy(ctx)

    assert chunks > tiles * 8, (chunks, tiles)
    assert R2 == R
    assert torch.equal(radii2, radii)
    assert torch.equal(color2.view(torch.int32), color.view(torch.int32))
    assert float(want["fragile"].double().mean()) <= FRAGILE_MAX
    errs = br.grad_errors(grads, br.blend_backward(*args, dL))
    assert all(e <= 1.0 for e in errs.values()), errs
