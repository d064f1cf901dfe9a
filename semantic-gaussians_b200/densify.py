"""Adaptive density control and optimiser bookkeeping of the 3DGS training loop: what
consumes ``viewspace_points.grad`` and ``radii`` produced by the rasterizer (train.py:158-175).

Behavioural contract: model/gaussian_model.py:196-240 (training_setup), :242-248 (update_learning_rate),
:283-286 (reset_opacity), :420-612 (prune / concatenate with Adam state, clone, split, densify_and_prune,
add_densification_stats) and utils/general_utils.py:32-63 (log-linear learning-rate schedule).  Written as one
table-driven mixin instead of the reference's per-attribute code; device-agnostic (the reference hard-codes
``device="cuda"``), so the logic is also covered by CPU tests."""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch
from torch import nn

# optimiser group name -> attribute of the model (model/gaussian_model.py:202-232)
GROUPS = (("xyz", "_xyz"), ("f_dc", "_features_dc"), ("f_rest", "_features_rest"), ("opacity", "_opacity"),
          ("scaling", "_scaling"), ("rotation", "_rotation"))
# Per-Gaussian tables outside the geometry: the semantic feature field (an optimiser group "semantic" when training
# arguments carry semantic_feature_lr) and the fusion view counts.  Whenever one has a row per Gaussian, densification
# keeps it row-aligned: clones and split children copy the parent's feature row and start with _times 0, pruned rows
# go.  A table without a row per Gaussian (empty, as a fresh model has them) is left as it is.
ROW_TABLES = (("semantic", "_features_semantic"), ("times", "_times"))


def expon_lr(lr_init: float, lr_final: float, max_steps: int, delay_steps: int = 0, delay_mult: float = 1.0
             ) -> Callable[[int], float]:
    """Log-linear interpolation from lr_init (step 0) to lr_final (step max_steps), optionally eased in by a
    sine ramp from delay_mult*lr to lr over delay_steps (utils/general_utils.py:32-63)."""
    def at(step: int) -> float:
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        ease = 1.0
        if delay_steps > 0:
            ease = delay_mult + (1.0 - delay_mult) * math.sin(0.5 * math.pi * min(max(step / delay_steps, 0.0), 1.0))
        t = min(max(step / max_steps, 0.0), 1.0)
        return ease * math.exp((1.0 - t) * math.log(lr_init) + t * math.log(lr_final))
    return at


class DensifyMixin:
    """Mixed into GaussianModel.  State: ``optimizer`` (Adam, one group per row of GROUPS, plus "semantic" when the
    feature field is trained), ``xyz_gradient_accum`` (P,1), ``denom`` (P,1), ``max_radii2D`` (P,),
    ``percent_dense``, ``spatial_lr_scale``.  Groups of other names (a decoder's weights) may share the optimiser:
    densification leaves them alone."""

    # ---- set-up -----------------------------------------------------------------------------------------
    def training_setup(self, training_args) -> None:
        dev = self._xyz.device
        P = self._xyz.shape[0]
        self.percent_dense = training_args.percent_dense
        self.xyz_gradient_accum = torch.zeros((P, 1), device=dev)
        self.denom = torch.zeros((P, 1), device=dev)
        if getattr(self, "max_radii2D", None) is None or self.max_radii2D.shape[0] != P:
            self.max_radii2D = torch.zeros((P,), device=dev)
        scale = getattr(self, "spatial_lr_scale", 1.0)
        lrs = {"xyz": training_args.position_lr_init * scale, "f_dc": training_args.feature_lr,
               "f_rest": training_args.feature_lr / 20.0, "opacity": training_args.opacity_lr,
               "scaling": training_args.scaling_lr, "rotation": training_args.rotation_lr}
        groups = []
        for name, attr in GROUPS:
            p = nn.Parameter(getattr(self, attr).detach().clone().requires_grad_(True))
            setattr(self, attr, p)
            groups.append({"params": [p], "lr": lrs[name], "name": name})
        semantic_lr = getattr(training_args, "semantic_feature_lr", None)
        if semantic_lr is not None and self._row_table("_features_semantic") is not None:
            p = nn.Parameter(self._features_semantic.detach().clone().requires_grad_(True))
            self._features_semantic = p
            groups.append({"params": [p], "lr": semantic_lr, "name": "semantic"})
        optimizer_type = getattr(training_args, "optimizer_type", "default")
        if optimizer_type == "default":
            self.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
        elif optimizer_type == "sparse_adam":  # 3DGS's name: step(visibility=...) leaves unseen Gaussians alone
            from .optim import GaussianAdam
            self.optimizer = GaussianAdam([dict(g, row_sparse=True) for g in groups], lr=0.0, eps=1e-15)
        else:
            raise ValueError(f"optimizer_type must be 'default' or 'sparse_adam', got {optimizer_type!r}")
        self._xyz_lr = expon_lr(training_args.position_lr_init * scale, training_args.position_lr_final * scale,
                                training_args.position_lr_max_steps, delay_mult=training_args.position_lr_delay_mult)

    def update_learning_rate(self, iteration: int) -> Optional[float]:
        for g in self.optimizer.param_groups:
            if g["name"] == "xyz":
                g["lr"] = self._xyz_lr(iteration)
                return g["lr"]
        return None

    def oneupSHdegree(self) -> None:
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    # ---- the one primitive: rewrite every parameter (and its Adam moments) row-wise ---------------------------
    def _row_table(self, attr: str) -> Optional[torch.Tensor]:
        """The ROW_TABLES entry ``attr`` if it has one row per Gaussian, else None."""
        t = getattr(self, attr, None)
        if isinstance(t, torch.Tensor) and t.ndim >= 1 and t.numel() > 0 and t.shape[0] == self._xyz.shape[0]:
            return t
        return None

    def _rewrite(self, rows: Callable[[str, torch.Tensor], torch.Tensor],
                 moments: Callable[[str, torch.Tensor], torch.Tensor]) -> None:
        """Replace each per-Gaussian group's parameter by ``rows(name, old)`` and, where Adam already holds moments
        for it, those by ``moments(name, m)``; re-bind the model attributes to the new Parameters.  The ROW_TABLES
        entries with a row per Gaussian that no group holds get ``rows(name, old)`` too; other groups are untouched."""
        attr_of = dict(GROUPS + ROW_TABLES)
        tables = [(n, a) for n, a in ROW_TABLES if self._row_table(a) is not None]  # before _xyz changes length
        for g in self.optimizer.param_groups:
            name = g.get("name")
            if name not in attr_of:
                continue
            old = g["params"][0]
            state = self.optimizer.state.pop(old, None)
            new = nn.Parameter(rows(name, old.detach()).requires_grad_(True))
            if state is not None:
                state["exp_avg"] = moments(name, state["exp_avg"])
                state["exp_avg_sq"] = moments(name, state["exp_avg_sq"])
                self.optimizer.state[new] = state
            g["params"][0] = new
            setattr(self, attr_of[name], new)
            tables = [(n, a) for n, a in tables if n != name]
        for name, attr in tables:
            old = getattr(self, attr)
            new = rows(name, old.detach())
            if isinstance(old, nn.Parameter):
                new = nn.Parameter(new, requires_grad=old.requires_grad)
            elif old.requires_grad:
                new.requires_grad_(True)
            setattr(self, attr, new)

    def prune_points(self, mask: torch.Tensor) -> None:
        """Remove the Gaussians where ``mask`` is True (gaussian_model.py:452-468)."""
        keep = ~mask
        self._rewrite(lambda _, t: t[keep], lambda _, m: m[keep])
        self.xyz_gradient_accum = self.xyz_gradient_accum[keep]
        self.denom = self.denom[keep]
        self.max_radii2D = self.max_radii2D[keep]

    def _append(self, new: Dict[str, torch.Tensor]) -> None:
        """Concatenate new Gaussians (zero Adam moments) and reset the statistics (gaussian_model.py:470-527).
        ``new`` holds the GROUPS rows and, for the ROW_TABLES the model has, their rows."""
        self._rewrite(lambda n, t: torch.cat((t, new[n]), dim=0),
                      lambda n, m: torch.cat((m, torch.zeros_like(new[n])), dim=0))
        P, dev = self._xyz.shape[0], self._xyz.device
        self.xyz_gradient_accum = torch.zeros((P, 1), device=dev)
        self.denom = torch.zeros((P, 1), device=dev)
        self.max_radii2D = torch.zeros((P,), device=dev)

    def replace_tensor_to_optimizer(self, tensor: torch.Tensor, name: str) -> Dict[str, torch.Tensor]:
        """Swap one per-Gaussian parameter for ``tensor`` with zeroed moments (gaussian_model.py:420-433).  A name
        that is not a per-Gaussian group changes nothing and returns {}."""
        attr_of = dict(GROUPS + ROW_TABLES)
        out = {}
        for g in self.optimizer.param_groups:
            if g.get("name") != name or name not in attr_of:
                continue
            old = g["params"][0]
            state = self.optimizer.state.pop(old, None)
            new = nn.Parameter(tensor.detach().clone().requires_grad_(True))
            if state is not None:
                state["exp_avg"] = torch.zeros_like(new)
                state["exp_avg_sq"] = torch.zeros_like(new)
                self.optimizer.state[new] = state
            g["params"][0] = new
            setattr(self, attr_of[name], new)
            out[name] = new
        return out

    def reset_opacity(self) -> None:
        """Clamp every opacity to at most 0.01 (gaussian_model.py:283-286)."""
        op = torch.minimum(self.get_opacity, torch.full_like(self.get_opacity, 0.01))
        self.replace_tensor_to_optimizer(torch.log(op / (1 - op)), "opacity")

    def _new_table_rows(self, parent_rows: Callable[[torch.Tensor], torch.Tensor]) -> Dict[str, torch.Tensor]:
        """Rows of the ROW_TABLES the model has for Gaussians made from ``parent_rows(table)``: the feature field
        copies the parents' rows, the view counts start at zero."""
        out = {}
        for name, attr in ROW_TABLES:
            t = self._row_table(attr)
            if t is not None:
                rows = parent_rows(t.detach())
                out[name] = torch.zeros_like(rows) if name == "times" else rows
        return out

    # ---- statistics + densification --------------------------------------------------------------------------
    def add_densification_stats(self, viewspace_point_tensor: torch.Tensor, update_filter: torch.Tensor) -> None:
        """Accumulate the screen-space positional gradient norm of the visible Gaussians (gaussian_model.py:608-612).
        The rasterizer delivers dL/dmean2D in the reference's units (pixel gradient x 0.5*W / 0.5*H)."""
        g = viewspace_point_tensor.grad[update_filter, :2]
        self.xyz_gradient_accum[update_filter] += torch.norm(g, dim=-1, keepdim=True)
        self.denom[update_filter] += 1

    def densify_and_clone(self, grads: torch.Tensor, grad_threshold: float, scene_extent: float) -> int:
        """Duplicate small Gaussians with a large positional gradient (gaussian_model.py:563-586)."""
        small = self.get_scaling.max(dim=1).values <= self.percent_dense * scene_extent
        sel = (torch.norm(grads, dim=-1) >= grad_threshold) & small
        new = {name: getattr(self, attr).detach()[sel] for name, attr in GROUPS}
        self._append(dict(new, **self._new_table_rows(lambda t: t[sel])))
        return int(sel.sum())

    def densify_and_split(self, grads: torch.Tensor, grad_threshold: float, scene_extent: float, N: int = 2) -> int:
        """Replace large Gaussians with a large positional gradient by N samples of themselves, each 1/(0.8 N)
        the size (gaussian_model.py:529-561).  ``grads`` covers the Gaussians that existed before cloning."""
        from .gaussian_model import build_rotation
        P, dev = self._xyz.shape[0], self._xyz.device
        padded = torch.zeros((P,), device=dev)
        padded[: grads.shape[0]] = grads.squeeze(-1) if grads.ndim > 1 else grads
        sel = (padded >= grad_threshold) & (self.get_scaling.max(dim=1).values > self.percent_dense * scene_extent)
        k = int(sel.sum())
        stds = self.get_scaling[sel].detach().repeat(N, 1)
        samples = torch.normal(mean=torch.zeros_like(stds), std=stds)
        rots = build_rotation(self._rotation.detach()[sel]).repeat(N, 1, 1)
        rep = lambda t: t.detach()[sel].repeat(N, *([1] * (t.ndim - 1)))
        self._append({
            "xyz": torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + rep(self._xyz),
            "f_dc": rep(self._features_dc), "f_rest": rep(self._features_rest), "opacity": rep(self._opacity),
            "scaling": torch.log(self.get_scaling[sel].detach().repeat(N, 1) / (0.8 * N)),
            "rotation": rep(self._rotation), **self._new_table_rows(rep)})
        self.prune_points(torch.cat((sel, torch.zeros(N * k, dtype=torch.bool, device=dev))))
        return k

    def densify_and_prune(self, max_grad: float, min_opacity: float, extent: float, max_screen_size) -> Dict[str, int]:
        """gaussian_model.py:588-606.  Returns the counts (cloned, split, pruned) for logging."""
        grads = self.xyz_gradient_accum / self.denom
        grads[grads.isnan()] = 0.0
        cloned = self.densify_and_clone(grads, max_grad, extent)
        split = self.densify_and_split(grads, max_grad, extent)
        prune = (self.get_opacity < min_opacity).squeeze(-1)
        if max_screen_size:
            prune = prune | (self.max_radii2D > max_screen_size) | (self.get_scaling.max(dim=1).values > 0.1 * extent)
        self.prune_points(prune)
        return {"cloned": cloned, "split": split, "pruned": int(prune.sum())}
