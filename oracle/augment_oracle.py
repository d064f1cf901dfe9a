"""numpy restatement of the elastic-distortion lookup (dataset/augmentation.py ElasticDistortion, the
``RegularGridInterpolator(ax, noise, bounds_error=0, fill_value=0)`` call as scipy 1.18 evaluates it), written as
``sgb_elastic_displace`` computes it: per axis the cell i with g[i] <= x < g[i+1] (the last cell at x == g[-1]),
t = (x - g[i]) / (g[i+1] - g[i]), the 8 corners in itertools.product order with weight ((1 * w0) * w1) * w2
summed from 0, 0 outside the grid, NaN for a NaN coordinate, then x + value * magnitude.  numpy rounds every
elementwise product and sum alone, as the kernel does.  Used by the tests as the checker of the device path and by
tools/time_distill.py as the host baseline."""
from __future__ import annotations

import random

import numpy as np


def lookup(xyz: np.ndarray, noise: np.ndarray, axes, magnitude: float) -> np.ndarray:
    """(P,3) fp64 ``xyz + interp(xyz) * magnitude`` for the (nx,ny,nz,3) fp32 ``noise`` on the three ``axes``."""
    x = np.asarray(xyz).astype(np.float64)
    P = x.shape[0]
    outside = np.zeros(P, bool)
    nan = np.isnan(x).any(axis=1)
    cell, t = [], []
    with np.errstate(invalid="ignore"):
        for a in range(3):
            g = np.asarray(axes[a]).astype(np.float64)
            outside |= (x[:, a] < g[0]) | (x[:, a] > g[-1])
            i = np.clip(np.searchsorted(g, x[:, a], side="right") - 1, 0, len(g) - 2)
            cell.append(i)
            t.append((x[:, a] - g[i]) / (g[i + 1] - g[i]))
        u = [1 - ta for ta in t]
        value = np.zeros((P, 3))
        for c in range(8):
            b = ((c >> 2) & 1, (c >> 1) & 1, c & 1)
            w = np.ones(P)
            for a in range(3):
                w = w * (t[a] if b[a] else u[a])
            corner = noise[cell[0] + b[0], cell[1] + b[1], cell[2] + b[2]].astype(np.float64)
            value = value + corner * w[:, None]
        value[outside] = 0.0
        value[nan] = np.nan
        return x + value * magnitude


def elastic_distortion(coords: np.ndarray, granularity: float, magnitude: float):
    """One distortion pass on the host: the noise from ``feature_dataset.noise_grid`` (numpy / scipy, drawing from
    ``np.random``) and ``lookup``.  Returns (distorted (P,3) fp64, noise_dim)."""
    from semantic_gaussians_b200.feature_dataset import noise_grid
    noise, ax = noise_grid(coords.min(0), coords.max(0), granularity)
    return lookup(coords, noise, ax, magnitude), noise.shape[:3]


def elastic_distortion_all(coords: np.ndarray, params):
    """``ElasticDistortion(params)(coords)``: the 0.95 gate from ``random``, then one pass per (granularity,
    magnitude).  Returns (coords, [noise_dim per pass])."""
    dims = []
    if random.random() < 0.95:
        for granularity, magnitude in params:
            coords, d = elastic_distortion(coords, granularity, magnitude)
            dims.append(d)
    return coords, dims
