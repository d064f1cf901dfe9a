"""CPU: sgb_adam_step's argument checks (they run before any CUDA call), optim.GaussianAdam on CPU tensors against
torch.optim.Adam and oracle/adam_oracle.py, its state_dict, and training_setup(optimizer_type=...) with the
moment bookkeeping of density control."""
import copy
import ctypes as C
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from adam_check import assert_step_matches_oracle  # noqa: E402
from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.densify import GROUPS  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.optim import GaussianAdam, visible_rows  # noqa: E402

SHAPES = [(50,), (40, 1), (33, 3), (21, 4), (17, 15, 3), (9, 48), (5, 256), (3, 513)]


# ---- C ABI ------------------------------------------------------------------------------------------------------
def _tensor(**kw):
    base = dict(param=16, grad=16, exp_avg=16, exp_avg_sq=16, visible=None, rows=10, row_len=4, beta1=0.9,
                beta2=0.999, eps=1e-8, step_size=1e-3, bias_correction2_sqrt=0.5)
    base.update(kw)
    return _lib.AdamTensor(**base)


def test_adam_step_is_exported():
    assert "sgb_adam_step" in _lib.EXPORTS and hasattr(_lib.load(), "sgb_adam_step")


@pytest.mark.parametrize("kw,msg", [
    (dict(param=None), b"null param"), (dict(grad=None), b"null grad"), (dict(exp_avg=None), b"null exp_avg"),
    (dict(exp_avg_sq=None), b"null exp_avg_sq"), (dict(rows=-1), b"rows"), (dict(row_len=0), b"row_len"),
    (dict(rows=0, row_len=-3), b"row_len"),
    (dict(beta1=1.0), b"beta1"), (dict(beta1=-0.1), b"beta1"), (dict(beta2=1.0), b"beta2"),
    (dict(beta2=float("nan")), b"beta2"), (dict(eps=-1e-8), b"eps"), (dict(step_size=float("inf")), b"step_size"),
    (dict(step_size=float("nan")), b"step_size"), (dict(bias_correction2_sqrt=0.0), b"bias_correction2_sqrt"),
    (dict(bias_correction2_sqrt=1.5), b"bias_correction2_sqrt"),
])
def test_invalid_tensor_is_rejected_before_cuda(kw, msg):
    lib = _lib.load()
    arr = (_lib.AdamTensor * 2)(_tensor(rows=0, param=None, grad=None, exp_avg=None, exp_avg_sq=None), _tensor(**kw))
    assert lib.sgb_adam_step(arr, 2, None) == -1
    err = lib.sgb_last_error()
    assert msg in err and b"tensor 1" in err


def test_invalid_count_and_null_array_are_rejected_and_empty_calls_launch_nothing():
    lib = _lib.load()
    arr = (_lib.AdamTensor * 1)(_tensor())
    assert lib.sgb_adam_step(arr, -1, None) == -1 and b"n = -1" in lib.sgb_last_error()
    assert lib.sgb_adam_step(arr, _lib.ADAM_MAX_TENSORS + 1, None) == -1 and b"n = 9" in lib.sgb_last_error()
    assert lib.sgb_adam_step(None, 1, None) == -1 and b"null tensors" in lib.sgb_last_error()
    # nothing to do: returns before any CUDA call, so also without a device
    assert lib.sgb_adam_step(None, 0, None) == 0
    empty = (_lib.AdamTensor * 1)(_tensor(rows=0, param=None, grad=None, exp_avg=None, exp_avg_sq=None))
    assert lib.sgb_adam_step(empty, 1, None) == 0


def test_struct_layout_matches_the_header():
    assert C.sizeof(_lib.AdamTensor) == 88 and _lib.AdamTensor.beta1.offset == 56 and _lib.AdamTensor.step_size.offset == 80


# ---- GaussianAdam on CPU tensors ----------------------------------------------------------------------------------
def _tables(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g)) for s in SHAPES]


def _set_grads(params, gen, scale=1.0):
    for p in params:
        p.grad = torch.randn(p.shape, generator=gen) * scale


def test_all_visible_matches_torch_adam():
    mine, ref = _tables(), _tables()
    a = GaussianAdam([{"params": mine[:4], "row_sparse": True}, {"params": mine[4:], "lr": 3e-3}], lr=1e-2, eps=1e-15)
    b = torch.optim.Adam([{"params": ref[:4]}, {"params": ref[4:], "lr": 3e-3}], lr=1e-2, eps=1e-15)
    gen = torch.Generator().manual_seed(1)
    for it in range(30):
        _set_grads(mine, gen)
        for p, q in zip(mine, ref):
            q.grad = p.grad.clone()
        a.step()
        b.step()
    for p, q in zip(mine, ref):
        torch.testing.assert_close(p, q, rtol=1e-6, atol=0)
        for k in ("exp_avg", "exp_avg_sq"):
            torch.testing.assert_close(a.state[p][k], b.state[q][k], rtol=1e-6, atol=0)
        assert float(a.state[p]["step"]) == float(b.state[q]["step"]) == 30
        assert a.state[p]["step"].dtype == b.state[q]["step"].dtype and a.state[p]["step"].device.type == "cpu"


@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.uint8])
def test_random_masks_leave_masked_rows_bitwise_and_match_the_oracle(mask_dtype):
    P = 64
    gen = torch.Generator().manual_seed(2)
    shapes = [(P,), (P, 3), (P, 15, 3), (P, 48), (P, 100)]
    params = [torch.nn.Parameter(torch.randn(s, generator=gen)) for s in shapes]
    dense = torch.nn.Parameter(torch.randn((7, 5), generator=gen))
    lr, betas, eps = 2e-2, (0.9, 0.999), 1e-8
    opt = GaussianAdam([{"params": params, "row_sparse": True}, {"params": [dense]}], lr=lr, betas=betas, eps=eps)
    for it in range(1, 9):
        _set_grads(params + [dense], gen)
        vis = torch.rand(P, generator=gen) < (0.0 if it == 4 else 0.4)
        for p in params:
            p.grad[~vis] = float("nan")                       # never read
        before = [(p.detach().numpy().copy(), p.grad.numpy().copy(),
                   opt.state[p]["exp_avg"].numpy().copy() if opt.state[p] else np.zeros(p.shape, np.float32),
                   opt.state[p]["exp_avg_sq"].numpy().copy() if opt.state[p] else np.zeros(p.shape, np.float32))
                  for p in params + [dense]]
        opt.step(visibility=vis.to(mask_dtype))
        for p, b in zip(params + [dense], before):
            st = opt.state[p]
            after = (p.detach().numpy(), st["exp_avg"].numpy(), st["exp_avg_sq"].numpy())
            assert_step_matches_oracle(b, after, it, lr, betas, eps, visible=None if p is dense else vis.numpy())


def test_parameter_without_grad_is_skipped():
    a, b = torch.nn.Parameter(torch.ones(4, 3)), torch.nn.Parameter(torch.ones(4, 3))
    opt = GaussianAdam([a, b], lr=0.1)
    a.grad = torch.ones_like(a)
    opt.step()
    assert torch.equal(b, torch.ones(4, 3)) and b not in opt.state and float(opt.state[a]["step"]) == 1
    assert float(a.detach()[0, 0]) == pytest.approx(0.9, rel=1e-6)


def test_state_dict_round_trip_and_exchange_with_torch_adam():
    gen = torch.Generator().manual_seed(3)
    mine, ref = _tables(4), _tables(4)
    a = GaussianAdam([{"params": mine, "row_sparse": False}], lr=1e-2)
    b = torch.optim.Adam(ref, lr=1e-2)
    for _ in range(3):
        _set_grads(mine, gen)
        a.step()
    # with itself
    mine2 = [torch.nn.Parameter(p.detach().clone()) for p in mine]
    a2 = GaussianAdam([{"params": mine2, "row_sparse": False}], lr=1e-2)
    a2.load_state_dict(copy.deepcopy(a.state_dict()))
    # to torch.optim.Adam: the per-parameter state under torch's own group options
    for p, q in zip(mine, ref):
        q.data.copy_(p.data)
    sd = b.state_dict()
    sd["state"] = copy.deepcopy(a.state_dict()["state"])
    b.load_state_dict(sd)
    _set_grads(mine, gen)
    for p, p2, q in zip(mine, mine2, ref):
        p2.grad, q.grad = p.grad.clone(), p.grad.clone()
    a.step(), a2.step(), b.step()
    for p, p2, q in zip(mine, mine2, ref):
        assert torch.equal(p, p2) and torch.equal(a.state[p]["exp_avg_sq"], a2.state[p2]["exp_avg_sq"])
        torch.testing.assert_close(p, q, rtol=1e-6, atol=0)
        assert float(b.state[q]["step"]) == 4
    # and back: torch's state into a fresh GaussianAdam
    mine3 = [torch.nn.Parameter(q.detach().clone()) for q in ref]
    a3 = GaussianAdam(mine3, lr=1e-2)
    sd = a3.state_dict()
    sd["state"] = copy.deepcopy(b.state_dict()["state"])
    a3.load_state_dict(sd)
    _set_grads(ref, gen)
    for q, p3 in zip(ref, mine3):
        p3.grad = q.grad.clone()
    b.step(), a3.step()
    for q, p3 in zip(ref, mine3):
        torch.testing.assert_close(p3, q, rtol=1e-6, atol=0)
        assert float(a3.state[p3]["step"]) == 5


def test_argument_errors():
    with pytest.raises(ValueError, match="weight_decay"):
        GaussianAdam([torch.nn.Parameter(torch.zeros(3))], weight_decay=0.1)
    with pytest.raises(ValueError, match="amsgrad"):
        GaussianAdam([{"params": [torch.nn.Parameter(torch.zeros(3))], "amsgrad": True}])
    half = torch.nn.Parameter(torch.zeros(4, 2, dtype=torch.float16))
    half.grad = torch.zeros_like(half)
    with pytest.raises(ValueError, match="float32"):
        GaussianAdam([half]).step()
    nc = torch.nn.Parameter(torch.zeros(4, 6).t())
    nc.grad = torch.zeros(6, 4)
    assert not nc.is_contiguous()
    with pytest.raises(ValueError, match="contiguous"):
        GaussianAdam([nc]).step()
    p = torch.nn.Parameter(torch.zeros(5, 3))
    p.grad = torch.ones_like(p)
    opt = GaussianAdam([{"params": [p], "row_sparse": True}])
    with pytest.raises(ValueError, match="length 4"):
        opt.step(visibility=torch.ones(4, dtype=torch.bool))
    with pytest.raises(ValueError, match="bool or uint8"):
        opt.step(visibility=torch.ones(5, dtype=torch.float32))
    with pytest.raises(ValueError, match="bool or uint8"):
        opt.step(visibility=torch.ones((5, 1), dtype=torch.bool))
    with pytest.raises(ValueError, match="visibility is on"):
        opt.step(visibility=torch.ones(5, dtype=torch.bool, device="meta"))
    assert torch.equal(p.detach(), torch.zeros(5, 3))       # no failed call moved the parameter


def test_visible_rows_is_the_union_over_views():
    a = {"visibility_filter": torch.tensor([True, False, False, True])}
    b = {"visibility_filter": torch.tensor([False, False, True, True])}
    assert visible_rows(a) is a["visibility_filter"]
    assert visible_rows([a, b]).tolist() == [True, False, True, True]
    with pytest.raises(ValueError):
        visible_rows([])


# ---- training_setup and density control -------------------------------------------------------------------------
ARGS = dict(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
            position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=0.05, scaling_lr=5e-3, rotation_lr=1e-3)


def _model(P=200, seed=0, **extra):
    g = torch.Generator().manual_seed(seed)
    scales = torch.exp(torch.randn(P, 3, generator=g) * 0.8 - 3.0)
    rot = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=1)
    m = GaussianModel.from_activated(torch.randn(P, 3, generator=g), scales, rot, torch.rand(P, generator=g) * 0.9 + 0.05,
                                     shs=torch.randn(P, 16, 3, generator=g), device="cpu")
    m.spatial_lr_scale = 2.0
    m.training_setup(SimpleNamespace(**ARGS, **extra))
    return m


def _step(m, visibility=None):
    loss = sum((getattr(m, a) ** 2).sum() for _, a in GROUPS)
    loss.backward()
    if visibility is None:
        m.optimizer.step()
    else:
        m.optimizer.step(visibility=visibility)
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


def test_training_setup_selects_the_optimizer():
    for m in (_model(), _model(optimizer_type="default")):
        assert type(m.optimizer) is torch.optim.Adam
        assert [g["name"] for g in m.optimizer.param_groups] == [n for n, _ in GROUPS]
        assert m.optimizer.defaults["eps"] == 1e-15 and m.optimizer.defaults["lr"] == 0.0
        assert all("row_sparse" not in g for g in m.optimizer.param_groups)
    s = _model(optimizer_type="sparse_adam")
    assert type(s.optimizer) is GaussianAdam
    ref = _model()
    for gs, gr in zip(s.optimizer.param_groups, ref.optimizer.param_groups):
        assert gs["name"] == gr["name"] and gs["lr"] == gr["lr"] and gs["eps"] == 1e-15 and gs["row_sparse"] is True
        assert gs["betas"] == gr["betas"]
    assert math.isclose(s.update_learning_rate(30000), 1.6e-6 * 2.0)
    with pytest.raises(ValueError, match="optimizer_type"):
        _model(optimizer_type="adamw")


def test_sparse_adam_step_moves_only_visible_gaussians():
    m = _model(optimizer_type="sparse_adam")
    before = {a: getattr(m, a).detach().clone() for _, a in GROUPS}
    vis = torch.zeros(200, dtype=torch.bool)
    vis[::4] = True
    _step(m, vis)
    for _, a in GROUPS:
        now = getattr(m, a).detach()
        assert torch.equal(now[~vis], before[a][~vis]) and not torch.equal(now[vis], before[a][vis])
        st = m.optimizer.state[getattr(m, a)]
        assert float(st["exp_avg"][~vis].abs().max()) == 0.0 and float(st["exp_avg_sq"][vis].min()) >= 0.0


def test_sparse_adam_prune_keeps_moments_of_survivors():
    m = _model(optimizer_type="sparse_adam")
    _step(m)
    before = {n: (getattr(m, a).detach().clone(), m.optimizer.state[getattr(m, a)]["exp_avg"].clone()) for n, a in GROUPS}
    mask = torch.zeros(200, dtype=torch.bool)
    mask[::3] = True
    m.prune_points(mask)
    _consistent(m)
    for n, a in GROUPS:
        assert torch.equal(getattr(m, a).detach(), before[n][0][~mask])
        assert torch.equal(m.optimizer.state[getattr(m, a)]["exp_avg"], before[n][1][~mask])
    _step(m, ~mask[~mask])                                   # a step through the rewritten parameters
    _consistent(m)


def test_sparse_adam_clone_split_append_and_reset_opacity():
    torch.manual_seed(0)
    m = _model(300, 1, optimizer_type="sparse_adam")
    _step(m)
    vs = torch.zeros(300, 3, requires_grad=True)
    vs.grad = torch.zeros(300, 3)
    vs.grad[:150, 0] = 1.0
    vis = torch.zeros(300, dtype=torch.bool)
    vis[:200] = True
    m.add_densification_stats(vs, vis)
    small = m.get_scaling.max(dim=1).values.detach() <= ARGS["percent_dense"] * 5.0
    n_clone = int(small[:150].sum())
    n_split = 150 - n_clone
    out = m.densify_and_prune(0.5, 0.0, 5.0, None)
    assert out == {"cloned": n_clone, "split": n_split, "pruned": 0}
    P = 300 + n_clone + n_split
    assert m._xyz.shape[0] == P
    _consistent(m)
    nk = 300 - n_split
    ea = m.optimizer.state[m._xyz]["exp_avg"]
    assert float(ea[nk:].abs().max()) == 0.0 and float(ea[:nk].abs().max()) > 0.0     # new rows start from zero
    m.reset_opacity()
    assert float(m.get_opacity.max()) <= 0.01 + 1e-7
    st = m.optimizer.state[m._opacity]
    assert float(st["exp_avg"].abs().max()) == 0.0 and float(st["exp_avg_sq"].abs().max()) == 0.0
    assert float(st["step"]) == 1
    _consistent(m)
    seen = torch.rand(P) < 0.5
    _step(m, seen)
    _consistent(m)
    assert float(m.optimizer.state[m._opacity]["exp_avg"][~seen].abs().max()) == 0.0
    assert float(m.optimizer.state[m._opacity]["step"]) == 2
