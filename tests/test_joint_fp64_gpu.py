"""The joint render (sgb_forward_render_joint_batch / sgb_backward_joint_batch: RGB from SH and a c-channel feature
table over one geometry state and one binning per view) against the float64 restatements, with anti-aliasing off
and on.  For c > 4 the alpha pass that builds the feature image's weight pool is also the RGB blend (it accumulates
colour, median depth and E / A in the same walk), so the RGB image is checked here in every branch that walk takes:

  c = 1, 3, 4, 5, 17, 64, 257 .. the small-C blend (c <= 4) and the weight pool + chain / dL/dfeature kernels
  opaque ....................... early termination
  dense_faint .................. weight-pool overflow and retry (the retry builds the pool without the RGB part,
                                 so the RGB image must survive from the first walk)
  w161 / w162 / w163, 13x7, 1x64  ragged and one-pixel-wide images
  sparse ....................... empty and one-entry tiles
  batch_empty_middle ........... V = 3 with a middle view that sees nothing
  grads_offset4 ................ dL_dcolors and dL_dfeatures 4 bytes off 16-byte alignment
  exp_alpha .................... E / A and their upstream gradients (the geometry restatement is skipped: their
                                 dL/dz lives in ctx scratch, test_depth_alpha_gpu.py covers it)
  fresh_backward_ctx ........... the backward on a ctx that does not hold the forward's weight pool: it is rebuilt
                                 by a plain alpha pass

Checked per view (tests/raster_check.py): RGB, the feature image, E / A, final_T, n_contrib, the summed blend
gradients dL_dmeans2D / dL_dconic / dL_dopacity, the RGB dL_dcolors, dL_dfeatures summed over the views, and (without
E / A) every geometry output and gradient.  Tolerances are blend_ref's and geom_ref's, unchanged."""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from raster_check import assert_ok, check_views, report  # noqa: E402

from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu

# name: (P, W, H, c, scale_mean, opacity or None, check_views keywords)
CASES = {f"c{c}": (20000, 160, 96, c, 0.02, None, {}) for c in (1, 3, 4, 5, 17, 64, 257)}
CASES.update({
    "opaque": (4000, 160, 96, 32, 0.08, 0.999, {}),
    "dense_faint": (100000, 128, 96, 65, 0.05, 0.02, {}),
    "w161": (20000, 161, 96, 32, 0.02, None, {}),
    "w162": (20000, 162, 96, 32, 0.02, None, {}),
    "w163": (20000, 163, 96, 32, 0.02, None, {}),
    "tile_13x7": (20000, 13, 7, 32, 0.02, None, {}),
    "one_pixel_wide": (20000, 1, 64, 32, 0.02, None, {}),
    "sparse": (150, 160, 96, 32, 0.02, None, {}),
    "batch_empty_middle": (20000, 160, 96, 17, 0.02, None, {}),
    "grads_offset4": (20000, 160, 96, 64, 0.02, None, dict(dcolors_offset=4)),
    "exp_alpha": (20000, 160, 96, 64, 0.02, None, dict(exp_alpha=True)),
    "fresh_backward_ctx": (20000, 160, 96, 64, 0.02, None, dict(fresh_backward_ctx=True)),
})


@pytest.mark.parametrize("aa", [False, True], ids=["aa_off", "aa_on"])
@pytest.mark.parametrize("name", list(CASES))
def test_joint_matches_fp64(name, aa):
    P, W, H, c, scale, opacity, kw = CASES[name]
    scene = make_scene(P, seed=42, sh=True, scale_mean=scale)
    if opacity is not None:
        scene.opacity[:] = opacity
    feats = np.random.default_rng(5).standard_normal((P, c)).astype(np.float32)
    bgf = np.linspace(-0.5, 0.5, c).astype(np.float32)
    cams = [orbit_cameras(4, W, H)[1]]
    if name == "batch_empty_middle":
        cams = orbit_cameras(3, W, H)
        cams[1] = look_at_camera((3.0, 0.0, 0.4), (6.0, 0.0, 0.4), W, H)   # looks away from the scene: R = 0
    t0 = time.time()
    res = check_views(scene, cams, np.array([0.2, 0.4, 0.6], np.float32), sh_degree=3, joint=(feats, bgf),
                      antialiasing=aa, seed=3, **kw)
    report("joint", f"{name} aa={int(aa)}", res, t0)
    assert_ok(res)
    assert "features" in res["errs"] and "dL_dfeatures" in res["errs"]
    if kw.get("exp_alpha"):
        assert "exp_alpha" in res["errs"]
    else:
        assert "dL_dmeans3D" in res["errs"]
    L = res["lens"]
    if name == "sparse":
        assert int((L == 0).sum()) > 0 and int((L == 1).sum()) > 0
    if name == "opaque":
        tile = torch.arange(H * W) // W // 16 * ((W + 15) // 16) + torch.arange(H * W) % W // 16
        assert float((res["n_contrib"] < L[tile] // 2).double().mean()) > 0.5
    if name == "dense_faint":
        assert int((L > 512).sum()) > 0
        assert res["chunks"] > L.numel() * 8      # the first guess of 8 chunks per tile overflowed and was retried
    if name == "batch_empty_middle":
        assert len(res["radii"]) == 3 and int(res["radii"][1].max()) == 0
