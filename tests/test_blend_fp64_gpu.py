"""The blend kernels against the float64 restatement (tests/blend_ref.py), through the C ABI, at every channel
count, image shape, list length and pointer layout the kernels branch on.  The restatement runs on the kernel's own
per-Gaussian state and tile lists (sgb_state_field), so the only error measured is the kernel's arithmetic.

Which case reaches which branch (C <= 4: blend_fwd.cu / blend_bwd.cu; C > 4: weight_pool.cu + chn_*.cu):
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
  feat_offset4 ............... feature rows not 16-byte aligned with C % 4 == 0: blend_forward_ldg_kernel and
                               chain_backward_warp_kernel<false>
  dcolors_offset4 ............ dL_dcolors not 16-byte aligned: red16 off
  zero_bg .................... the bg_nonzero == 0 branch of the chain kernel (C = 17, 64, 257)
  batch, batch_empty_middle .. sgb_*_batch with V = 3 views and one shared dL_dcolors; a middle view with R = 0
  calibration ................ the configurations test_parity_gpu.py::test_backward_vs_reference pins to the
                               compiled reference
test_parity_gpu.py::test_channel_forward_and_backward_above_65535_tiles checks tile rows 254-256 of a 257 x 257
tile image (tile ids across 65535) with check_views() (tests/raster_check.py), which
also checks every view's geometry stage against tests/geom_ref.py."""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from raster_check import assert_ok as _assert_ok, check_views, report  # noqa: E402

from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu


def _report(name, res, t0):
    report("blend", name, res, t0)


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
