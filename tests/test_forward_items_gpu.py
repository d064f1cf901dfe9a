"""The forward C-channel contraction (blend_forward_persistent_kernel) against the float64 restatement
(tests/blend_ref.py) on what its (tile, up to 128 channels) work items branch on:
  C = 5, 17, 64, 127, 128 ....... one item per tile; channel groups past the item idle, a lane's last group masked
  C = 129, 255, 256, 257 ........ two or three items per tile (80 + 49, 128 + 127, 128 + 128, 96 + 96 + 65)
  C = 384, 512 .................. three and four 128-channel items
  entry counts .................. tiles of exactly 0, 1, 15, 16, 17, 127, 128, 129, 255, 256, 257 and 300 entries:
                                  empty tiles, partial and full ring stages, ring wrap and multi-chunk tiles
  W = 193 ....................... a ragged last tile: scalar stores in the epilogue
  feat_offset4 .................. a feature table that is not 16-byte aligned: rows staged by the producer warp
  C = 17 ........................ C % 4 != 0: rows staged by the producer warp, zero-filled past the item
and the non-finite repair of a feature row whose only non-finite channel lies in the second item.  The scene is
test_dfeature_items_gpu.py's: each tile's Gaussians are tiny, faint and inside the tile, so the tile's list length is
its weight-pool entry count."""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from raster_check import assert_ok, check_views, report  # noqa: E402
from test_dfeature_items_gpu import COUNTS, _check_counts, placed_scene  # noqa: E402
from util import dev_cam, dev_scene, run_ours  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = {f"c{C}": (C, 192, {}) for C in (5, 17, 64, 127, 128, 129, 255, 256, 257, 384, 512)}
CASES.update({
    "c256_w193": (256, 193, {}),
    "c129_w193": (129, 193, {}),
    "c256_feat_offset4": (256, 192, dict(feat_offset=4)),
    "c17_feat_offset4": (17, 192, dict(feat_offset=4)),
})


@pytest.mark.parametrize("name", list(CASES))
def test_forward_items_match_fp64(name):
    C, W, layout = CASES[name]
    scene, cam = placed_scene(C, W)
    bg = np.linspace(0.05, 0.5, C).astype(np.float32)
    t0 = time.time()
    res = check_views(scene, [cam], bg, **layout)
    report("forward", name, res, t0)
    assert_ok(res)
    _check_counts(res["lens"], W)


def _render(scene, cam, bg):
    dev = torch.device("cuda:0")
    out = run_ours("chn", dev_scene(scene, dev), dev_cam(cam, dev), torch.as_tensor(bg, device=dev),
                   use_features=True)["color"]
    torch.cuda.synchronize()
    return out.detach().clone()


def test_nonfinite_channel_in_second_item():
    """A feature row that is non-finite in channel 200 only (the second 128-channel item at C = 256) reaches exactly
    the pixels that blend its Gaussian, in exactly that channel; every other value is bitwise that of a run with the
    row made finite."""
    C, W, ch = 256, 192, 200
    scene, cam = placed_scene(C, W)
    g = sum(COUNTS[:6]) + 3   # a Gaussian of the 128-entry tile (eight full ring stages)
    assert COUNTS[6] == 128
    bg = np.linspace(0.05, 0.5, C).astype(np.float32)
    finite = _render(scene, cam, bg)
    # where the Gaussian is blended: its weight, read back as channel ch of a scene whose only non-zero feature is it
    marker = scene.features.copy()
    scene.features = np.zeros_like(marker)
    scene.features[g, ch] = 1.0
    blended = _render(scene, cam, np.zeros(C, np.float32))[ch] != 0
    scene.features = marker.copy()
    scene.features[g, ch] = np.inf
    bad = _render(scene, cam, bg)
    assert 0 < int(blended.sum()) < blended.numel() // 10, int(blended.sum())

    nonfinite = ~torch.isfinite(bad)
    assert torch.equal(nonfinite[ch], blended)
    others = torch.ones_like(nonfinite)
    others[ch] = False
    assert not bool(nonfinite[others].any())
    # pixels that do not blend the Gaussian, every channel: bit for bit
    keep = ~blended.unsqueeze(0).expand_as(bad)
    assert torch.equal(bad[keep].view(torch.int32), finite[keep].view(torch.int32))
    # pixels that do, every other channel: bit for bit as well
    hit = blended.unsqueeze(0).expand_as(bad) & others
    assert torch.equal(bad[hit].view(torch.int32), finite[hit].view(torch.int32))
