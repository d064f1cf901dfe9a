"""Adam for the per-Gaussian parameter tables: one native launch per step for up to eight tables, and rows a view
did not see are left alone (csrc/adam.cu, ``sgb_adam_step``)."""
from __future__ import annotations

import math
from typing import Iterable, Optional, Union

import torch

from . import _lib


def visible_rows(outs: Union[dict, Iterable[dict]]) -> torch.Tensor:
    """The (P,) bool mask of the Gaussians at least one view saw: the OR of ``out["visibility_filter"]`` over one
    render output or a list of them (``render_batch`` / ``render_chn_batch``).  What a step over those views passes
    as ``GaussianAdam.step(visibility=...)``."""
    if isinstance(outs, dict):
        return outs["visibility_filter"]
    outs = list(outs)
    if not outs:
        raise ValueError("visible_rows needs at least one render output")
    vis = outs[0]["visibility_filter"]
    for o in outs[1:]:
        vis = vis | o["visibility_filter"]
    return vis


class GaussianAdam(torch.optim.Optimizer):
    """``torch.optim.Adam`` (no ``amsgrad``, ``weight_decay``, ``maximize``) whose CUDA step is one kernel launch for
    up to eight parameters, each element read and written once, with an optional per-Gaussian visibility mask.

    Groups take the option ``row_sparse`` (default ``False``): the first dimension of the group's parameters is the
    Gaussian index.  ``step(visibility=mask)`` then updates only the rows of those parameters where ``mask`` is set;
    of every other row nothing is read or written, so the parameter and both moments stay bitwise as they were and a
    non-finite gradient there is never seen.  The moments of an unseen row therefore neither decay nor move the row:
    dense Adam would keep pushing it along its stale momentum.  Groups that are not ``row_sparse`` (a decoder's
    weight and bias) always step densely, and ``visibility=None`` steps everything.

    This is the rule of 3DGS's ``optimizer_type="sparse_adam"``, with one difference: that optimizer drops Adam's
    bias corrections and this one keeps them.  ``state[p]["step"]`` is the parameter's global step count as in
    ``torch.optim.Adam`` (a row does not count its own visits), so with every row visible the update is
    ``torch.optim.Adam``'s up to rounding.  The per-parameter state has torch's keys and representation
    (``step``, ``exp_avg``, ``exp_avg_sq``): the ``"state"`` part of a ``state_dict()`` carries over to a
    ``torch.optim.Adam`` over the same parameters and back.

    Parameters and gradients are contiguous fp32.  CUDA parameters go through ``sgb_adam_step`` (bias corrections
    computed on the host in double; nothing synchronises); CPU parameters take the same update as torch expressions.
    """

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, **unsupported):
        if unsupported:
            raise ValueError(f"GaussianAdam does not take {sorted(unsupported)} (plain Adam: lr, betas, eps and the "
                             "group option row_sparse)")
        if not 0.0 <= lr:
            raise ValueError(f"invalid learning rate {lr}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"invalid betas {betas}")
        if not 0.0 <= eps:
            raise ValueError(f"invalid eps {eps}")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, row_sparse=False))

    def add_param_group(self, param_group: dict) -> None:
        bad = set(param_group) & {"weight_decay", "amsgrad", "maximize", "capturable", "foreach", "fused",
                                  "differentiable"}
        if bad:
            raise ValueError(f"GaussianAdam does not take the group options {sorted(bad)}")
        super().add_param_group(param_group)

    @staticmethod
    def _mask(visibility: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        if visibility is None:
            return None
        if not isinstance(visibility, torch.Tensor) or visibility.ndim != 1 or \
                visibility.dtype not in (torch.bool, torch.uint8):
            raise ValueError("visibility must be a 1-D bool or uint8 tensor with one entry per Gaussian")
        v = visibility.detach().contiguous()
        return v.view(torch.uint8) if v.dtype == torch.bool else v

    @torch.no_grad()
    def step(self, visibility: Optional[torch.Tensor] = None, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        vis = self._mask(visibility)
        native = {}                                                # device -> [AdamTensor]
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                if p.dtype != torch.float32 or g.dtype != torch.float32:
                    raise ValueError(f"GaussianAdam needs float32 parameters and gradients, got {p.dtype} / {g.dtype}")
                if g.is_sparse or not p.is_contiguous() or not g.is_contiguous():
                    raise ValueError("GaussianAdam needs dense, contiguous parameters and gradients")
                mask = vis if group["row_sparse"] else None
                if mask is not None:
                    if p.ndim == 0 or p.shape[0] != mask.shape[0]:
                        raise ValueError(f"row_sparse parameter of shape {tuple(p.shape)} against a visibility mask of "
                                         f"length {mask.shape[0]}")
                    if mask.device != p.device:
                        raise ValueError(f"visibility is on {mask.device}, the parameter on {p.device}")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                m, v = state["exp_avg"], state["exp_avg_sq"]
                for t in (m, v):
                    if t.shape != p.shape or t.dtype != torch.float32 or t.device != p.device or not t.is_contiguous():
                        raise ValueError("exp_avg / exp_avg_sq must be contiguous float32 of the parameter's shape, on "
                                         "its device")
                if state["step"].device.type != "cpu":             # state loaded from a fused / capturable Adam
                    state["step"] = state["step"].cpu()
                state["step"] += 1
                t_ = float(state["step"])
                step_size = group["lr"] / (1.0 - beta1 ** t_)
                bc2_sqrt = math.sqrt(1.0 - beta2 ** t_)
                if p.numel() == 0:
                    continue
                if p.is_cuda:
                    rows = p.shape[0] if p.ndim > 0 else 1
                    native.setdefault(p.device, []).append(_lib.AdamTensor(
                        p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(),
                        mask.data_ptr() if mask is not None else None, rows, p.numel() // rows,
                        beta1, beta2, group["eps"], step_size, bc2_sqrt))
                elif mask is None:
                    _adam_update(p, g, m, v, beta1, beta2, group["eps"], step_size, bc2_sqrt)
                else:
                    idx = mask.nonzero().squeeze(1)
                    pi, mi, vi = p[idx], m[idx], v[idx]
                    _adam_update(pi, g[idx], mi, vi, beta1, beta2, group["eps"], step_size, bc2_sqrt)
                    p.index_copy_(0, idx, pi)
                    m.index_copy_(0, idx, mi)
                    v.index_copy_(0, idx, vi)
        for device, tensors in native.items():
            lib = _lib.load()
            with torch.cuda.device(device):
                stream = torch.cuda.current_stream(device).cuda_stream
                for i in range(0, len(tensors), _lib.ADAM_MAX_TENSORS):
                    chunk = tensors[i:i + _lib.ADAM_MAX_TENSORS]
                    _lib.check(lib.sgb_adam_step((_lib.AdamTensor * len(chunk))(*chunk), len(chunk), stream),
                               "sgb_adam_step")
        return loss


def _adam_update(p, g, m, v, beta1, beta2, eps, step_size, bc2_sqrt) -> None:
    """In place, the operations of torch.optim.Adam's single-tensor path."""
    m.lerp_(g, 1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    p.addcdiv_(m, (v.sqrt() / bc2_sqrt).add_(eps), value=-step_size)
