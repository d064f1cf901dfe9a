"""CPU: adaptive density control + optimiser bookkeeping (model/gaussian_model.py:196-248, 420-612)."""
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from semantic_gaussians_b200.densify import GROUPS, expon_lr
from semantic_gaussians_b200.gaussian_model import GaussianModel

ARGS = SimpleNamespace(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                       position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=0.05, scaling_lr=5e-3, rotation_lr=1e-3)


def _model(P=200, seed=0):
    g = torch.Generator().manual_seed(seed)
    scales = torch.exp(torch.randn(P, 3, generator=g) * 0.8 - 3.0)
    rot = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=1)
    m = GaussianModel.from_activated(torch.randn(P, 3, generator=g), scales, rot, torch.rand(P, generator=g) * 0.9 + 0.05,
                                     shs=torch.randn(P, 16, 3, generator=g), device="cpu")
    m.spatial_lr_scale = 2.0
    m.training_setup(ARGS)
    return m


def _step(m):
    """one fake optimisation step so that Adam holds moments"""
    loss = sum((getattr(m, a) ** 2).sum() for _, a in GROUPS)
    loss.backward()
    m.optimizer.step()
    m.optimizer.zero_grad(set_to_none=True)


def _consistent(m):
    P = m._xyz.shape[0]
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        assert p is getattr(m, dict(GROUPS)[g["name"]]) and p.shape[0] == P and p.requires_grad
        st = m.optimizer.state.get(p)
        if st is not None:
            assert st["exp_avg"].shape == p.shape and st["exp_avg_sq"].shape == p.shape
    assert m.xyz_gradient_accum.shape == (P, 1) and m.denom.shape == (P, 1) and m.max_radii2D.shape == (P,)
    assert len(m.optimizer.state) <= len(GROUPS)


def test_lr_schedule_matches_reference_formula():
    f = expon_lr(1e-2, 1e-4, 1000, delay_mult=0.01)
    assert math.isclose(f(0), 1e-2) and math.isclose(f(1000), 1e-4) and math.isclose(f(5000), 1e-4)
    assert math.isclose(f(500), math.exp(0.5 * math.log(1e-2) + 0.5 * math.log(1e-4)))
    g = expon_lr(1e-2, 1e-4, 1000, delay_steps=100, delay_mult=0.1)
    assert math.isclose(g(0), 0.1 * 1e-2) and math.isclose(g(50), (0.1 + 0.9 * math.sin(0.25 * math.pi)) * f(50))
    assert expon_lr(0.0, 0.0, 10)(3) == 0.0 and f(-1) == 0.0


def test_setup_groups_and_lr():
    m = _model()
    lrs = {g["name"]: g["lr"] for g in m.optimizer.param_groups}
    assert math.isclose(lrs["xyz"], 1.6e-4 * 2.0) and math.isclose(lrs["f_rest"], 2.5e-3 / 20) and lrs["opacity"] == 0.05
    assert m.optimizer.defaults["eps"] == 1e-15
    assert math.isclose(m.update_learning_rate(30000), 1.6e-6 * 2.0)
    _consistent(m)


def test_prune_keeps_moments_of_survivors():
    m = _model()
    _step(m)
    before = {n: (getattr(m, a).detach().clone(), m.optimizer.state[getattr(m, a)]["exp_avg"].clone()) for n, a in GROUPS}
    mask = torch.zeros(200, dtype=torch.bool)
    mask[::3] = True
    m.max_radii2D = torch.arange(200.0)
    m.prune_points(mask)
    _consistent(m)
    for n, a in GROUPS:
        assert torch.equal(getattr(m, a).detach(), before[n][0][~mask])
        assert torch.equal(m.optimizer.state[getattr(m, a)]["exp_avg"], before[n][1][~mask])
    assert torch.equal(m.max_radii2D, torch.arange(200.0)[~mask])


def test_clone_split_prune_counts_and_geometry():
    torch.manual_seed(0)
    m = _model(300, 1)
    _step(m)
    extent = 5.0
    vs = torch.zeros(300, 3, requires_grad=True)
    vs.grad = torch.zeros(300, 3)
    vs.grad[:150, 0] = 1.0                                  # large screen-space gradient on the first half
    vis = torch.zeros(300, dtype=torch.bool)
    vis[:200] = True
    m.add_densification_stats(vs, vis)
    assert float(m.denom.sum()) == 200 and float(m.xyz_gradient_accum[:150].min()) == 1.0
    scal = m.get_scaling.max(dim=1).values.detach()
    small = scal <= ARGS.percent_dense * extent
    n_clone = int((small[:150]).sum())
    n_split = 150 - n_clone
    assert n_clone > 0 and n_split > 0
    xyz0, sc0 = m._xyz.detach().clone(), m.get_scaling.detach().clone()
    out = m.densify_and_prune(0.5, 0.0, extent, None)      # min_opacity 0: nothing pruned by opacity
    assert out == {"cloned": n_clone, "split": n_split, "pruned": 0}
    assert m._xyz.shape[0] == 300 + n_clone + 2 * n_split - n_split
    _consistent(m)
    # originals that were split are gone, clones are exact copies, split children are 1/1.6 the size
    kept = torch.ones(300, dtype=torch.bool)
    kept[:150] = small[:150]
    nk = int(kept.sum())
    assert torch.equal(m._xyz.detach()[:nk], xyz0[kept])
    clone_src = torch.nonzero(small[:150]).squeeze(1)
    assert torch.equal(m._xyz.detach()[nk:nk + n_clone], xyz0[clone_src])
    split_src = torch.nonzero(~small[:150]).squeeze(1)
    children = m.get_scaling.detach()[nk + n_clone:]
    assert torch.allclose(children, sc0[split_src].repeat(2, 1) / 1.6, rtol=1e-5)
    # new Gaussians start with zero moments, survivors keep theirs
    ea = m.optimizer.state[m._xyz]["exp_avg"]
    assert float(ea[nk:].abs().max()) == 0.0 and float(ea[:nk].abs().max()) > 0.0
    assert float(m.xyz_gradient_accum.abs().max()) == 0.0


def test_screen_size_and_opacity_pruning_and_reset():
    m = _model(100, 2)
    _step(m)
    m.xyz_gradient_accum[:] = 0
    m.denom[:] = 0                                           # 0/0 -> nan -> treated as 0 (gaussian_model.py:590)
    m.max_radii2D = torch.zeros(100)
    m.max_radii2D[:7] = 50.0
    op = m.get_opacity.detach().squeeze(1)
    big_ws = m.get_scaling.max(dim=1).values.detach() > 0.1 * 5.0
    # reference quirk kept: clone/split reset max_radii2D (densification_postfix, gaussian_model.py:527) before the
    # screen-size test reads it (:600), so that criterion never fires right after a densification
    expect = (op < 0.3) | big_ws
    out = m.densify_and_prune(1e9, 0.3, 5.0, 20)
    assert out["cloned"] == 0 and out["split"] == 0 and out["pruned"] == int(expect.sum())
    assert m._xyz.shape[0] == 100 - int(expect.sum())
    m.reset_opacity()
    assert float(m.get_opacity.max()) <= 0.01 + 1e-7
    st = m.optimizer.state[m._opacity]
    assert float(st["exp_avg"].abs().max()) == 0.0 and float(st["exp_avg_sq"].abs().max()) == 0.0
    _consistent(m)
    m.active_sh_degree = 0
    for _ in range(5):
        m.oneupSHdegree()
    assert m.active_sh_degree == 3


def test_sh_degree_schedule_starts_at_zero_like_the_reference():
    """model/gaussian_model.py:47 + train.py:118: a fresh model starts at SH degree 0 and oneupSHdegree() raises it
    (capped at max_sh_degree); constructors of already-fitted scenes activate every band."""
    import numpy as np
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    m = GaussianModel(3)
    assert m.active_sh_degree == 0 and m.max_sh_degree == 3
    seen = []
    for _ in range(5):
        m.oneupSHdegree()
        seen.append(m.active_sh_degree)
    assert seen == [1, 2, 3, 3, 3]
    rng = np.random.default_rng(0)
    fitted = GaussianModel.from_activated(rng.standard_normal((4, 3)), np.full((4, 3), 0.1), np.tile([1.0, 0, 0, 0], (4, 1)),
                                          np.full(4, 0.5), device="cpu")
    assert fitted.active_sh_degree == 3
