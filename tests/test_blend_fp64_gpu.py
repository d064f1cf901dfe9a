"""The blend kernels against the float64 restatement (tests/blend_ref.py), through the C ABI, at every channel
count, image shape, list length and pointer layout the kernels branch on.  The restatement runs on the kernel's own
per-Gaussian state and tile lists (sgb_state_field), so the only error measured is the kernel's arithmetic.

Which case reaches which branch (C <= 4: blend_fwd.cu / blend_bwd.cu; C > 4: blend_v3.cu):
  C = 1, 2, 4 ................ the C <= 4 feature path with colors_precomp
  C = 5 .. 768 ............... 16-channel slabs of the chain kernel and 64-channel items of the dL/dfeature kernel,
                               on both sides of every multiple of 16 and 64 (plain loads when C % 4 != 0)
  W % 4 = 1, 2, 3 ............ image rows without TMA (cp.async dL tiles, dl_slab_plain), scalar row paths
  H % 16 != 0, 13 x 7, 1 x 64 . partial tiles, an image of one partial tile, a one-pixel-wide image
  sparse ..................... empty tiles and one-entry tiles
  opaque ..................... early termination: n_contrib well below the list length
  dense_faint ................ lists of 2 600 - 13 000 entries: beyond kMetaCap = 512 cached entries, every
                               remainder R = 1..8 of the 128-entry dL/dfeature passes, weight pool overflow and
                               retry on a fresh ctx
  dl_offset4 ................. dL/dout 4 bytes off 16-byte alignment with W % 4 == 0: non-TMA dL paths
  feat_offset4 ............... feature rows not 16-byte aligned with C % 4 == 0: blend_forward_v3_kernel and
                               chain_backward_warp_kernel<false>
  dcolors_offset4 ............ dL_dcolors not 16-byte aligned: red16 off
  zero_bg .................... the bg_nonzero == 0 branch of the chain kernel (C = 17, 64, 257)
  batch, batch_empty_middle .. sgb_*_batch with V = 3 views and one shared dL_dcolors; a middle view with R = 0
  calibration ................ the configurations test_parity_gpu.py::test_backward_vs_reference pins to the
                               compiled reference
test_parity_gpu.py::test_channel_forward_and_backward_above_65535_tiles checks tile rows 254-256 of a 257 x 257
tile image (tile ids across 65535) with check_views() below."""
import ctypes as Ct
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blend_ref as br  # noqa: E402
from util import dev_cam, dev_scene  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu

FRAGILE_MAX = 0.02   # at most this fraction of pixels may be left out of the comparison
DEV = torch.device("cuda:0")


def read_state(lib, P, R, W, H, geom, binning, img):
    """The blend's inputs and forward state of one view, as the kernels left them."""
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    spec = dict(means2D=(torch.float32, (P, 2)), conic_opacity=(torch.float32, (P, 4)),
                point_list=(torch.int32, (max(R, 1),)), ranges=(torch.int32, (tiles, 2)),
                n_contrib=(torch.int32, (H * W,)), final_T=(torch.float32, (H * W,)))
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


def check_views(scene, cams, bg, *, dl_offset=0, feat_offset=0, dcolors_offset=0, tile_rows=None, seed=0):
    """Forward and backward of len(cams) views of `scene` (features as colors_precomp) in one sgb_*_batch call
    sequence on a fresh ctx, each view checked against the float64 restatement on its own state; dL/dout is
    random, zero at fragile pixels and, with tile_rows, outside those tile rows.  Returns per-case statistics:
    compare() of every output (<= 1 passes), fragile fraction, list lengths and the weight-pool chunks."""
    lib = _lib.load()
    W, H = cams[0].image_width, cams[0].image_height
    P, Cn = scene.features.shape
    V = len(cams)
    sc = dev_scene(scene, DEV)
    feats = _placed(sc["features"], feat_offset)
    bg = torch.as_tensor(bg, dtype=torch.float32, device=DEV)
    cms = [dev_cam(c, DEV) for c in cams]
    inp = _lib.ViewInputs(
        P=P, D=0, M=0, W=W, H=H, C=Cn, background=bg.data_ptr(), means3D=sc["means3D"].data_ptr(), shs=None,
        colors_precomp=feats.data_ptr(), opacities=sc["opacities"].data_ptr(), scales=sc["scales"].data_ptr(),
        scale_modifier=1.0, rotations=sc["rotations"].data_ptr(), cov3D_precomp=None, viewmatrix=None,
        projmatrix=None, campos=None, tan_fovx=0.0, tan_fovy=0.0, prefiltered=0, debug=0)
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
        views, dLs = [], []
        for v in range(V):
            R = Rs[v]
            if R == 0:
                views.append(None)
                dLs.append(torch.randn((Cn, H, W), device=DEV, generator=g))
                continue
            st = read_state(lib, P, R, W, H, geom[v], binning[v], img[v])
            args = (st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], sc["features"], bg, W, H)
            want = br.blend_forward(*args, tile_rows=tile_rows)
            dL = torch.randn((Cn, H * W), device=DEV, generator=g)
            dL[:, want["fragile"]] = 0.0
            if tile_rows is not None:
                dL[:, :tile_rows[0] * 16 * W] = 0.0
                dL[:, tile_rows[1] * 16 * W:] = 0.0
            views.append((st, args, want))
            dLs.append(dL.reshape(Cn, H, W))
        dL_in = [_placed(d, dl_offset) for d in dLs]
        z = lambda *s: torch.zeros(s, device=DEV)
        dcolors = _placed(z(P, Cn), dcolors_offset)
        grads = [dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 4), dL_dopacity=z(P), dL_dcolors=dcolors,
                      dL_dmeans3D=z(P, 3), dL_dcov3D=z(P, 6), dL_dscales=z(P, 3), dL_drotations=z(P, 4))
                 for _ in cams]
        gr = (_lib.ViewGrads * V)(*[_lib.ViewGrads(dL_dsh=None, **{k: t.data_ptr() for k, t in gv.items()})
                                    for gv in grads])
        _lib.check(lib.sgb_backward_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(radii), ptrs(geom), ptrs(binning),
                                          ptrs(img), ptrs(dL_in), gr, stream), "sgb_backward_batch")
    finally:
        torch.cuda.synchronize(DEV)
        lib.sgb_ctx_destroy(ctx)

    errs = {}
    frag, lens = [], []
    want_colors = torch.zeros((P, Cn), dtype=torch.float64, device=DEV)
    for v in range(V):
        if views[v] is None:   # nothing in view: the image is the background, no gradient
            assert torch.equal(color[v], bg[:, None, None].expand(Cn, H, W))
            for name in ("dL_dmeans2D", "dL_dconic", "dL_dopacity"):
                assert float(grads[v][name].abs().max()) == 0.0, name
            continue
        st, args, want = views[v]
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
        got_grads["dL_dcolors"] = wb["dL_dcolors"]   # the shared buffer is checked against the sum below
        e = dict(final_T=br.compare(st["final_T"][ok], want["final_T"][ok]),
                 color=br.compare(color[v].reshape(Cn, -1)[:, ok], want["color"].reshape(Cn, -1)[:, ok]))
        e.update({k: x for k, x in br.grad_errors(got_grads, wb).items() if k != "dL_dcolors"})
        for k, x in e.items():
            errs[k] = max(errs.get(k, 0.0), x)
        for name in ("dL_dmeans2D", "dL_dconic", "dL_dopacity"):
            assert float(wb[name].abs().max()) > 0, name
        rg = st["ranges"].long()
        lens.append(rg[:, 1] - rg[:, 0])
    errs["dL_dcolors"] = br.compare(dcolors, want_colors)
    assert float(want_colors.abs().max()) > 0
    return dict(errs=errs, fragile=max(frag), lens=torch.cat(lens).cpu(), chunks=chunks,
                n_contrib=views[0][0]["n_contrib"].cpu() if views[0] else None, W=W, H=H)


def _report(name, res, t0):
    e = " ".join(f"{k}={v:.3g}" for k, v in res["errs"].items())
    print(f"\n[fp64 blend] {name}: fragile={res['fragile']:.4%} {e} ({time.time() - t0:.1f} s)")


def _assert_ok(res):
    assert res["fragile"] <= FRAGILE_MAX, res["fragile"]
    assert all(v <= 1.0 for v in res["errs"].values()), res["errs"]


BG_RAMP = "ramp"


def _bg(kind, C):
    return np.zeros(C, np.float32) if kind == "zero" else np.linspace(0.05, 0.5, C).astype(np.float32)


# name: (P, W, H, C, scale_mean, opacity or None, background, layout offsets)
CASES = {f"c{C}": (20000, 160, 96, C, 0.02, None, BG_RAMP, {})
         for C in (1, 2, 4, 5, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 256, 257)}
CASES.update({
    "c768": (20000, 64, 48, 768, 0.02, None, BG_RAMP, {}),
    "c17_zero_bg": (20000, 160, 96, 17, 0.02, None, "zero", {}),
    "c64_zero_bg": (20000, 160, 96, 64, 0.02, None, "zero", {}),
    "c257_zero_bg": (20000, 160, 96, 257, 0.02, None, "zero", {}),
    "w161": (20000, 161, 96, 32, 0.02, None, BG_RAMP, {}),
    "w162": (20000, 162, 96, 32, 0.02, None, BG_RAMP, {}),
    "w163": (20000, 163, 96, 32, 0.02, None, BG_RAMP, {}),
    "h100": (20000, 160, 100, 32, 0.02, None, BG_RAMP, {}),
    "w161_c5": (20000, 161, 100, 5, 0.02, None, BG_RAMP, {}),
    "tile_13x7": (20000, 13, 7, 32, 0.02, None, BG_RAMP, {}),
    "one_pixel_wide": (20000, 1, 64, 32, 0.02, None, BG_RAMP, {}),
    "sparse": (300, 160, 96, 32, 0.02, None, BG_RAMP, {}),
    "opaque": (4000, 160, 96, 32, 0.08, 0.999, BG_RAMP, {}),
    "dense_faint_c16": (100000, 128, 96, 16, 0.05, 0.02, BG_RAMP, {}),
    "dense_faint_c65": (100000, 128, 96, 65, 0.05, 0.02, BG_RAMP, {}),
    "dl_offset4": (20000, 160, 96, 32, 0.02, None, BG_RAMP, dict(dl_offset=4)),
    "feat_offset4": (20000, 160, 96, 32, 0.02, None, BG_RAMP, dict(feat_offset=4)),
    "dcolors_offset4": (20000, 160, 96, 32, 0.02, None, BG_RAMP, dict(dcolors_offset=4)),
})


@pytest.mark.parametrize("name", list(CASES))
def test_blend_matches_fp64(name):
    P, W, H, C, scale, opacity, bgk, layout = CASES[name]
    scene = make_scene(P, seed=40, channels=C, scale_mean=scale)
    if opacity is not None:
        scene.opacity[:] = opacity
    t0 = time.time()
    res = check_views(scene, [orbit_cameras(4, W, H)[1]], _bg(bgk, C), **layout)
    _report(name, res, t0)
    _assert_ok(res)
    L = res["lens"]
    if name == "sparse":
        assert int((L == 0).sum()) > 0 and int((L == 1).sum()) > 0
    if name == "opaque":
        tile = torch.arange(H * W) // W // 16 * ((W + 15) // 16) + torch.arange(H * W) % W // 16
        assert float((res["n_contrib"] < L[tile] // 2).double().mean()) > 0.5
    if name.startswith("dense_faint"):
        big = L[L > 512]
        assert big.numel() > 0
        assert set((((big - 1) % 128) // 16 + 1).tolist()) == set(range(1, 9))   # every partial last pass
        assert res["chunks"] > L.numel() * 8      # the first guess of 8 chunks per tile overflowed and was retried


@pytest.mark.parametrize("C,empty_middle", [(64, False), (17, True)])
def test_batch_matches_fp64(C, empty_middle):
    W, H = 160, 96
    scene = make_scene(20000, seed=41, channels=C)
    cams = orbit_cameras(3, W, H)
    if empty_middle:   # looks away from the scene: R = 0
        cams[1] = look_at_camera((3.0, 0.0, 0.4), (6.0, 0.0, 0.4), W, H)
    t0 = time.time()
    res = check_views(scene, cams, _bg(BG_RAMP, C), seed=3)
    _report(f"batch C={C} empty_middle={empty_middle}", res, t0)
    _assert_ok(res)


@pytest.mark.parametrize("P,W,H,C", [(50000, 320, 240, 3), (50000, 320, 240, 100), (30000, 333, 211, 100),
                                     (100000, 640, 480, 256)])
def test_calibration_configurations_match_fp64(P, W, H, C):
    """The scenes, cameras and backgrounds of test_backward_vs_reference's feature cases, whose kernels are also
    pinned to the compiled reference: a failure here would mean the restatement or the tolerance is wrong."""
    scene = make_scene(P, seed=2, channels=C)
    t0 = time.time()
    res = check_views(scene, [orbit_cameras(4, W, H)[1]], np.linspace(0.0, 0.5, C).astype(np.float32), seed=5)
    _report(f"calibration P={P} {W}x{H} C={C}", res, t0)
    _assert_ok(res)
