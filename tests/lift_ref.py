"""The lift of feature maps onto the Gaussians (sgb_lift_batch) restated in float64 for the tests, on the front-to-back
walk of tests/blend_ref.py: per tile, feat_sum += w^T F and weight_sum += the sum of each entry's weights, with
w = alpha * T exactly as blend_ref._walk computes it.  Runs on CPU and CUDA tensors alike."""
from __future__ import annotations

import torch

from blend_ref import ALPHA_MIN, _f64, _tiles, _walk


def lift(means2D, conic_opacity, point_list, ranges, maps, W, H, tile_rows=None):
    """The lift of one view on the kernel's per-Gaussian state and tile lists: feat_sum (P, C) = w^T F per tile and
    weight_sum (P,) = the sum of each entry's weights over the tile's pixels, in float64; maps (C, H, W).  fragile
    (H W) is blend_ref.blend_forward's.  A test zeroes the map at fragile pixels, but weight_sum takes every pixel:
    weight_ok (P,) marks the Gaussians whose alpha stays below half the 1/255 cut at every fragile pixel, so that no
    fp32 decision there can give them a weight, and whose weight sums an fp32 kernel therefore reproduces to
    rounding."""
    dev = torch.as_tensor(means2D).device
    mean, con = _f64(means2D, dev).reshape(-1, 2), _f64(conic_opacity, dev).reshape(-1, 4)
    pl = torch.as_tensor(point_list).to(dev, torch.int64).reshape(-1)
    F = _f64(maps, dev).reshape(-1, H * W)
    P, C = mean.shape[0], F.shape[0]
    feat = torch.zeros((P, C), dtype=torch.float64, device=dev)
    wsum = torch.zeros(P, dtype=torch.float64, device=dev)
    fragile = torch.zeros(H * W, dtype=torch.bool, device=dev)
    reach = torch.zeros(P, dtype=torch.bool, device=dev)
    for _, s, e, px, py in _tiles(ranges, W, H, tile_rows):
        ids = pl[s:e]
        k = _walk(mean, con, ids, px, py)
        pix = (py * W + px).to(dev)
        feat.index_add_(0, ids, k["w"].T @ F[:, pix].T)
        wsum.index_add_(0, ids, k["w"].sum(0))
        fragile[pix] = k["fragile"]
        near = (k["op"] * k["G"] >= 0.5 * ALPHA_MIN) & k["fragile"][:, None]
        reach[ids[near.any(dim=0)]] = True
    return dict(feat_sum=feat, weight_sum=wsum, fragile=fragile, weight_ok=~reach)
