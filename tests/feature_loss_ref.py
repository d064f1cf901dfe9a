"""The reference's feature distillation loss (distill.py:111-124) as plain torch expressions in float64, restated for
the tests: the plane, decoded and voxel-row losses are all this loss on their own layout of rows."""
from __future__ import annotations

import torch


def feature_loss(x: torch.Tensor, y: torch.Tensor, loss_type: str):
    """x, y (rows, C), one row per pixel or voxel -> (loss, count, d loss / d x (rows, C)), all in float64 by
    autograd.  count is the number of rows the mean runs over: rows of y with a non-zero element for cosine, every row
    for l1 / l2.  With no row to average over the loss is 0 and the gradient zero (cosine: the reference skips such a
    batch)."""
    x = x.detach().double().requires_grad_(True)
    y = y.double()
    m = y.norm(dim=-1) > 0
    count = int(m.sum()) if loss_type == "cosine" else x.shape[0]
    if count == 0:
        return 0.0, 0, torch.zeros_like(x)
    if loss_type == "cosine":
        loss = (1 - torch.nn.CosineSimilarity()(x[m], y[m])).mean()
    elif loss_type == "l1":
        loss = torch.nn.L1Loss()(x, y)
    else:
        loss = torch.nn.MSELoss()(x, y)
    loss.backward()
    return float(loss.detach()), count, x.grad
