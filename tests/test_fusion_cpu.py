"""Fusion oracle (oracle/fusion_oracle.py) pinned against golden vectors produced by the
REFERENCE's own PointCloudToImageMapper + fusion.py accumulate statements
(tests/golden/make_fusion_golden.py)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_fusion_golden import fusion_inputs, other_seed_inputs  # noqa: E402
from make_raster_golden import digest  # noqa: E402

from oracle import fusion_oracle as fo  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fusion_golden.npz")


@pytest.fixture(scope="module")
def data():
    return fusion_inputs(), np.load(GOLD)


@pytest.mark.parametrize("mode", ["none", "surface", "depth"])
def test_mapping_and_fusion_match_reference(data, mode):
    (scene, cams, feats, depths), gold = data
    w, h = cams[0].image_width, cams[0].image_height
    P, C = scene.P, feats[0].shape[0]
    feat_sum = np.zeros((P, C), np.float32)
    count = np.zeros(P, np.float32)
    for i, cam in enumerate(cams):
        K = fo.rescale_intrinsics(cam.intrinsics(), [w, h])
        depth = {"none": None, "surface": "surface", "depth": depths[i]}[mode]
        m = fo.compute_mapping(cam.world_view_transform, scene.xyz, [w, h], K, 0.05, 4, depth)
        g = gold[f"{mode}_mapping_{i}"]
        assert m.dtype == np.int64 and m.shape == g.shape
        assert np.array_equal(m, g), f"view {i}: {(m != g).any(axis=1).sum()} rows differ"   # bit-exact indices
        fo.accumulate(feats[i], m, feat_sum, count)
    fo.normalize(feat_sum, count)
    assert np.array_equal(count.reshape(-1, 1), gold[f"{mode}_times"])
    assert np.array_equal(digest(feat_sum), gold[f"{mode}_fused.sha256"])   # same fp32 sums, same order


def test_some_points_visible_and_some_not(data):
    _, gold = data
    for mode in ("none", "surface", "depth"):
        vis = gold[f"{mode}_mapping_0"][:, 2]
        assert 0 < vis.sum() < vis.size


def test_oracle_matches_reference_on_other_seed(data):
    _, gold = data
    scene, cams, feats, depths = other_seed_inputs()
    for i, cam in enumerate(cams):
        for j, depth in enumerate((None, "surface", depths[i])):
            K = fo.rescale_intrinsics(cam.intrinsics(), [96, 64])
            got = fo.compute_mapping(cam.world_view_transform, scene.xyz, [96, 64], K, 0.1, 2, depth)
            assert np.array_equal(got, gold[f"other_mapping_{i}_{j}"])
