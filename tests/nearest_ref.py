"""Brute-force restatement of sgb_nearest (include/sgb200.h) for the tests: every query against every reference row,
in fp32, with the contract's expression d2 = (dx*dx + dy*dy) + dz*dz, dx = q.x - r.x.  Each torch elementwise op
rounds its result to fp32 on its own (no FMA contraction), so the oracle is the numpy float32 expression bit for bit,
and it runs on whichever device its inputs are on: on the GPU for the large cases."""
import numpy as np
import torch


def d2_numpy(q: np.ndarray, r: np.ndarray) -> np.ndarray:
    """(m, P) float32 d2 of every pair, the contract's expression in numpy."""
    dx = q[:, 0:1] - r[None, :, 0]
    dy = q[:, 1:2] - r[None, :, 1]
    dz = q[:, 2:3] - r[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def nearest_oracle(query: torch.Tensor, ref: torch.Tensor, max_dist2: float = float("inf"), chunk: int = 1 << 26):
    """(index int64 (M,), dist2 float32 (M,)) of sgb_nearest for float32 (M,3) / (P,3) tensors on one device."""
    M, P = query.shape[0], ref.shape[0]
    dev = query.device
    index = torch.full((M,), -1, dtype=torch.int64, device=dev)
    dist2 = torch.full((M,), float("inf"), dtype=torch.float32, device=dev)
    if M == 0 or P == 0:
        return index, dist2
    limit = torch.tensor(max_dist2, dtype=torch.float32, device=dev)
    rfin = torch.isfinite(ref).all(1)
    qfin = torch.isfinite(query).all(1)
    cols = torch.arange(P, device=dev)
    inf = torch.tensor(float("inf"), device=dev)
    step = max(1, chunk // P)
    for s in range(0, M, step):
        q = query[s:s + step]
        dx = q[:, 0:1] - ref[None, :, 0]
        dy = q[:, 1:2] - ref[None, :, 1]
        dz = q[:, 2:3] - ref[None, :, 2]
        d = (dx * dx + dy * dy) + dz * dz
        ok = rfin[None] & qfin[s:s + step, None] & (d <= limit)
        best = torch.where(ok, d, inf).amin(1)
        j = torch.where(ok & (d == best[:, None]), cols[None], P).amin(1)     # smallest row among the minima
        has = j < P
        index[s:s + step] = torch.where(has, j, -1)
        dist2[s:s + step] = torch.where(has, best, inf)
    return index, dist2
