"""The dL/dfeature contraction (dfeature_persistent_kernel<T>) against the float64 restatements (tests/blend_ref.py for
a backward, tests/lift_ref.py for an fp16 lift) on what its (tile, up to 256 channels) work items branch on:
  C = 5, 64, 255, 256 ........... one item per tile, narrower than 256 channels below 256 (idle compute warps)
  C = 257, 512 .................. two items per tile (144 + 113 channels; 256 + 256)
  entry counts .................. tiles of exactly 0, 1, 15, 16, 17, 127, 128, 129, 255, 256, 257 and 300 entries: the
                                  R = ceil(cnt / 16) specialisation, a pass boundary on both sides, three passes
  fp16 dL ....................... the lift's half-precision map through the same items
  W % 4 != 0 .................... dL slabs staged by the producer warp (cp.async fp32, plain loads fp16)
  dcolors_offset4 ............... dL_dcolors not 16-byte aligned: scalar reductions
Each tile's Gaussians are tiny, faint and placed inside the tile, so every binned Gaussian touches its tile and the
tile's list length is its weight-pool entry count."""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from raster_check import assert_ok, check_views, report  # noqa: E402
from test_lift_gpu import F16, F32, check_lift  # noqa: E402

from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene  # noqa: E402

pytestmark = pytest.mark.gpu

COUNTS = (0, 1, 15, 16, 17, 127, 128, 129, 255, 256, 257, 300)   # entries of tile 0, 1, ... of a one-tile-row image


def _pixel(cam, xyz):
    """Pixel coordinates (the rasterizer's ndc2Pix) of world points (N, 3)."""
    proj = np.asarray(cam.full_proj_transform, np.float64).reshape(4, 4)
    h = np.concatenate([xyz, np.ones((xyz.shape[0], 1))], 1) @ proj
    ndc = h[:, :2] / h[:, 3:4]
    return np.stack([((ndc[:, 0] + 1.0) * cam.image_width - 1.0) * 0.5,
                     ((ndc[:, 1] + 1.0) * cam.image_height - 1.0) * 0.5], 1)


def placed_scene(C, W, seed=0):
    """A scene and a camera of a W x 16 image whose tile t holds exactly COUNTS[t] Gaussians, each projected to a
    pixel 4..11 px inside its tile with a 2 px radius, opacity 0.05."""
    cam = look_at_camera((0.0, -3.0, 0.0), (0.0, 0.0, 0.0), W, 16)
    P = sum(COUNTS)
    scene = make_scene(P, seed=seed, channels=C)
    rng = np.random.default_rng(seed)
    tile = np.repeat(np.arange(len(COUNTS)), COUNTS)
    want = np.stack([tile * 16 + rng.integers(4, 12, P), rng.integers(4, 12, P)], 1).astype(np.float64)
    # view space -> world: the pixel is affine in (x / z, y / z) at a fixed depth
    view = np.asarray(cam.world_view_transform, np.float64).reshape(4, 4)
    to_world = lambda t: (t - view[3, :3]) @ np.linalg.inv(view[:3, :3])
    z = 3.0
    base = [to_world(np.array([[u * z, v * z, z]])) for u, v in ((0.0, 0.0), (0.1, 0.0), (0.0, 0.1))]
    p0, px, py = (_pixel(cam, b)[0] for b in base)
    A = np.stack([(px - p0) / 0.1, (py - p0) / 0.1], 1)
    uv = np.linalg.solve(A, (want - p0).T).T
    t = np.stack([uv[:, 0] * z, uv[:, 1] * z, np.full(P, z)], 1)
    scene.xyz[:] = to_world(t).astype(np.float32)
    assert np.abs(_pixel(cam, scene.xyz.astype(np.float64)) - want).max() < 1e-2
    scene.scales[:] = 0.002
    scene.opacity[:] = 0.05
    return scene, cam


def _check_counts(lens, W):
    tiles = (W + 15) // 16
    assert lens.tolist() == list(COUNTS) + [0] * (tiles - len(COUNTS))


CASES = {f"c{C}": (C, 192, {}) for C in (5, 64, 255, 256, 257, 512)}
CASES.update({
    "c256_w193": (256, 193, {}),
    "c257_dcolors_offset4": (257, 192, dict(dcolors_offset=4)),
    "c256_dcolors_offset4": (256, 192, dict(dcolors_offset=4)),
})


@pytest.mark.parametrize("name", list(CASES))
def test_dfeature_items_match_fp64(name):
    C, W, layout = CASES[name]
    scene, cam = placed_scene(C, W)
    bg = np.linspace(0.05, 0.5, C).astype(np.float32)
    t0 = time.time()
    res = check_views(scene, [cam], bg, **layout)
    report("dfeature", name, res, t0)
    assert_ok(res)
    _check_counts(res["lens"], W)


@pytest.mark.parametrize("C,W,dt", [(256, 192, F16), (512, 192, F16), (257, 192, F16), (256, 196, F16),
                                    (256, 193, F32)])
def test_dfeature_items_lift_matches_fp64(C, W, dt):
    scene, cam = placed_scene(1, W)
    res = check_lift(scene, [cam], C, dt)
    print(f"\n[lift fp64] C={C} W={W} {dt}: fragile={res['fragile']:.4%} " +
          " ".join(f"{k}={v:.3g}" for k, v in res["errs"].items()))
    assert res["fragile"] <= 0.02, res["fragile"]
    assert all(v <= 1.0 for v in res["errs"].values()), res["errs"]
    _check_counts(res["lens"], W)
