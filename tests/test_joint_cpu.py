"""CPU: densification keeps the semantic feature table and the view counts row-aligned with the Gaussians, trains the
table as an optimiser group, and leaves non-Gaussian groups (a decoder) alone; the joint render's argument checks."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from semantic_gaussians_b200.densify import GROUPS
from semantic_gaussians_b200.gaussian_model import GaussianModel
from semantic_gaussians_b200.optim import GaussianAdam

ARGS = dict(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
            position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=0.05, scaling_lr=5e-3, rotation_lr=1e-3)
EXTENT = 5.0


def _model(P=300, seed=1, semantic=None, **args):
    g = torch.Generator().manual_seed(seed)
    scales = torch.exp(torch.randn(P, 3, generator=g) * 0.8 - 3.0)
    rot = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=1)
    m = GaussianModel.from_activated(torch.randn(P, 3, generator=g), scales, rot, torch.rand(P, generator=g) * 0.9 + 0.05,
                                     shs=torch.randn(P, 16, 3, generator=g), device="cpu")
    m.spatial_lr_scale = 2.0
    if semantic is not None:
        m.create_semantic(semantic)
        m._features_semantic = torch.randn(P, semantic, generator=g)
        m._times = torch.rand(P, 1, generator=g) + 1.0
    m.training_setup(SimpleNamespace(**ARGS, **args))
    return m


def _step(m, extra=()):
    """one fake optimisation step so that Adam holds moments for every trained table"""
    tables = [getattr(m, a) for _, a in GROUPS] + list(extra)
    if any(g["name"] == "semantic" for g in m.optimizer.param_groups):
        tables.append(m._features_semantic)
    sum((t ** 2).sum() for t in tables).backward()
    m.optimizer.step()
    m.optimizer.zero_grad(set_to_none=True)


def _densify(m, seed=0):
    """First half of the Gaussians get a large screen-space gradient; densify_and_prune with an opacity threshold
    that prunes some.  Returns (clone parents, split parents, survivors among the originals, prune mask) in terms of
    the original rows, computed the way densify_and_prune decides."""
    P = m._xyz.shape[0]
    vs = torch.zeros(P, 3, requires_grad=True)
    vs.grad = torch.zeros(P, 3)
    vs.grad[: P // 2, 0] = 1.0
    m.add_densification_stats(vs, torch.ones(P, dtype=torch.bool))
    torch.manual_seed(seed)
    return m.densify_and_prune(0.5, 0.2, EXTENT, None)


def _split_rows(m):
    P = m._xyz.shape[0]
    small = m.get_scaling.max(dim=1).values.detach() <= ARGS["percent_dense"] * EXTENT
    big = torch.zeros(P, dtype=torch.bool)
    big[: P // 2] = True
    return torch.nonzero(big & small).squeeze(1), torch.nonzero(big & ~small).squeeze(1)


def _expected_rows(m, table, new_rows):
    """The row order densify_and_prune produces for a table: originals, clones, split children (N = 2), minus the
    split parents, then minus the opacity-pruned rows (which the caller applies)."""
    clone_src, split_src = _split_rows(m)
    P = table.shape[0]
    after_clone = torch.cat((table, new_rows(table[clone_src])))
    keep = torch.ones(after_clone.shape[0] + 2 * len(split_src), dtype=torch.bool)
    keep[split_src] = False
    return torch.cat((after_clone, new_rows(table[split_src].repeat(2, 1))))[keep]


@pytest.mark.parametrize("optimised", [False, True])
def test_feature_table_and_times_follow_the_rows(optimised):
    args = dict(semantic_feature_lr=1e-3) if optimised else {}
    m = _model(semantic=8, **args)
    _step(m)
    feats0, times0 = m._features_semantic.detach().clone(), m._times.detach().clone()
    xyz0 = m._xyz.detach().clone()
    names = [g["name"] for g in m.optimizer.param_groups]
    assert ("semantic" in names) == optimised
    op_before = m.get_opacity.detach().squeeze(1).clone()
    exp_feats = _expected_rows(m, feats0, lambda r: r)
    exp_times = _expected_rows(m, times0, torch.zeros_like)
    exp_xyz_keep = _expected_rows(m, xyz0, lambda r: r)
    exp_op = _expected_rows(m, op_before[:, None], lambda r: r).squeeze(1)
    out = _densify(m)
    assert out["cloned"] > 0 and out["split"] > 0 and out["pruned"] > 0
    keep = ~(exp_op < 0.2)
    P = m._xyz.shape[0]
    assert m._features_semantic.shape == (P, 8) and m._times.shape == (P, 1)
    assert torch.equal(m._features_semantic.detach(), exp_feats[keep])
    assert torch.equal(m._times.detach(), exp_times[keep])
    # the survivors among the originals and the clones are exact copies (split children are resampled)
    n_orig_clone = int(keep[: xyz0.shape[0] + out["cloned"] - out["split"]].sum())
    assert torch.equal(m._xyz.detach()[:n_orig_clone], exp_xyz_keep[keep][:n_orig_clone])
    if optimised:
        g = next(g for g in m.optimizer.param_groups if g["name"] == "semantic")
        assert g["params"][0] is m._features_semantic and m._features_semantic.requires_grad


@pytest.mark.parametrize("optimizer_type", ["default", "sparse_adam"])
def test_semantic_moments_kept_for_survivors_zero_for_new_rows(optimizer_type):
    m = _model(semantic=6, semantic_feature_lr=1e-3, optimizer_type=optimizer_type)
    g = next(g for g in m.optimizer.param_groups if g["name"] == "semantic")
    assert g["lr"] == 1e-3
    if optimizer_type == "sparse_adam":
        assert isinstance(m.optimizer, GaussianAdam) and g["row_sparse"]
    _step(m)
    st = m.optimizer.state[m._features_semantic]
    m0, v0 = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
    exp_m = _expected_rows(m, m0, torch.zeros_like)
    exp_v = _expected_rows(m, v0, torch.zeros_like)
    op = _expected_rows(m, m.get_opacity.detach(), lambda r: r).squeeze(1)
    _densify(m)
    keep = ~(op < 0.2)
    st = m.optimizer.state[m._features_semantic]
    assert torch.equal(st["exp_avg"], exp_m[keep]) and torch.equal(st["exp_avg_sq"], exp_v[keep])
    assert float(st["exp_avg"].abs().max()) > 0.0
    _step(m)  # the optimiser still steps the rewritten table


def test_decoder_group_is_left_alone():
    m = _model(semantic=4, semantic_feature_lr=1e-3)
    dec = torch.nn.Linear(4, 16)
    m.optimizer.add_param_group({"params": list(dec.parameters()), "lr": 1e-3, "name": "decoder"})
    m.optimizer.add_param_group({"params": [torch.nn.Parameter(torch.ones(3))], "lr": 1e-3})  # no name at all
    _step(m, extra=list(dec.parameters()))
    w, b = dec.weight, dec.bias
    w0, mw0 = w.detach().clone(), m.optimizer.state[w]["exp_avg"].clone()
    _densify(m)
    g = next(g for g in m.optimizer.param_groups if g.get("name") == "decoder")
    assert g["params"][0] is w and g["params"][1] is b
    assert torch.equal(w.detach(), w0) and torch.equal(m.optimizer.state[w]["exp_avg"], mw0)
    assert m.replace_tensor_to_optimizer(torch.zeros(16, 4), "decoder") == {}
    assert g["params"][0] is w
    m.reset_opacity()
    assert m._features_semantic.shape[0] == m._xyz.shape[0]


def test_without_semantic_table_nothing_changes():
    """Without a semantic table, semantic_feature_lr alone adds no group and changes no tensor: the optimiser holds the
    GROUPS only, and densification gives the same parameters and moments as a model trained without the argument.
    (The no-table path itself is tests/test_densify_cpu.py's.)"""
    a = _model(seed=3)
    b = _model(seed=3, semantic_feature_lr=1e-3)  # no table: the argument alone adds nothing
    for m in (a, b):
        assert [g["name"] for g in m.optimizer.param_groups] == [n for n, _ in GROUPS]
        _step(m)
        _densify(m, seed=7)
        assert m._features_semantic.numel() == 0 and m._times.numel() == 0
    for _, attr in GROUPS:
        assert torch.equal(getattr(a, attr).detach(), getattr(b, attr).detach())
        assert torch.equal(a.optimizer.state[getattr(a, attr)]["exp_avg"], b.optimizer.state[getattr(b, attr)]["exp_avg"])


def test_table_without_a_row_per_gaussian_is_left_alone():
    m = _model()
    m._features_semantic = torch.randn(5, 3)  # not one row per Gaussian: not the model's field
    _step(m)
    _densify(m)
    assert m._features_semantic.shape == (5, 3)


# ---- native argument checks: rejected before anything is enqueued, so they run without a device ------------------
def _lib_or_skip():
    from semantic_gaussians_b200 import _lib
    try:
        return _lib, _lib.load()
    except (ImportError, OSError) as e:
        pytest.skip(f"libsgb200.so not built: {e}")


def _inputs(_lib, buf, shs=False, C3=3):
    p = C.addressof(buf)
    return _lib.ViewInputs(P=10, D=0, M=1 if shs else 0, W=32, H=32, C=C3, background=p, means3D=p,
                           shs=p if shs else None, colors_precomp=None if shs else p, opacities=p, scales=p,
                           scale_modifier=1.0, rotations=p, cov3D_precomp=None, viewmatrix=p, projmatrix=p, campos=p,
                           tan_fovx=0.5, tan_fovy=0.5, prefiltered=0, debug=0)


def _fwd(lib, _lib, inp, feats, c, bg, exp=True, alpha=True):
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    arr = (C.c_void_p * 1)(p)
    cams = (_lib.Camera * 1)(_lib.Camera(p.value, p.value, p.value, 0.5, 0.5))
    R = (C.c_int64 * 1)(0)
    return lib.sgb_forward_render_joint_batch(1, C.byref(inp), 1, cams, R, arr, arr, arr, arr, arr, arr,
                                              arr if exp else None, arr if alpha else None, feats, c, bg, arr, None)


@pytest.mark.parametrize("case,msg", [
    ("null_features", b"feature table"), ("c0", b"c >= 1"), ("null_bg", b"feature background"),
    ("exp_without_alpha", b"together"), ("rgb_not_3", b"C = 3")])
def test_joint_forward_rejects_bad_arguments(case, msg):
    _lib, lib = _lib_or_skip()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    inp = _inputs(_lib, buf, C3=5 if case == "rgb_not_3" else 3)
    feats = None if case == "null_features" else p
    c = 0 if case == "c0" else 8
    bg = None if case == "null_bg" else p
    rc = _fwd(lib, _lib, inp, feats, c, bg, alpha=case != "exp_without_alpha")
    assert rc == -1 and msg in lib.sgb_last_error()


@pytest.mark.parametrize("case,msg", [("null_features", b"feature table"), ("c0", b"c >= 1"),
                                      ("shared_dL_dcolors", b"dL_dcolors"), ("null_dfeat", b"null")])
def test_joint_backward_rejects_bad_arguments(case, msg):
    _lib, lib = _lib_or_skip()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    V = 2
    inp = _inputs(_lib, buf, shs=True)
    arr = (C.c_void_p * V)(p, p)
    cams = (_lib.Camera * V)(*[_lib.Camera(p, p, p, 0.5, 0.5)] * V)
    R = (C.c_int64 * V)(1, 1)
    grads = (_lib.ViewGrads * V)(*[_lib.ViewGrads(*[p] * 9)] * V)  # every view the same dL_dcolors
    if case != "shared_dL_dcolors":
        grads[1].dL_dcolors = p + 64
    rc = lib.sgb_backward_joint_batch(1, C.byref(inp), V, cams, R, arr, arr, arr, arr, arr, None, None, grads,
                                      None if case == "null_features" else p, 0 if case == "c0" else 8, p,
                                      None if case == "null_dfeat" else arr, p, None)
    assert rc == -1 and msg in lib.sgb_last_error()
