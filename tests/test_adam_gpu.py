"""GPU: optim.GaussianAdam / sgb_adam_step (csrc/adam.cu) against oracle/adam_oracle.py at every row length its
kernel branches on, with dense, random and empty visibility masks; against torch.optim.Adam; launch count,
synchronisation and reproducibility; and inside the two training loops it is meant for."""
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
from semantic_gaussians_b200.optim import GaussianAdam, visible_rows  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
MAX_ORACLE_ROWS = 6000       # a table with more elements than MAX_ORACLE_ELEMS is compared on a sample of its rows
MAX_ORACLE_ELEMS = 2_000_000


def _rows_to_compare(rows, row_len, gen):
    if rows * row_len <= MAX_ORACLE_ELEMS:
        return None
    k = MAX_ORACLE_ROWS // 3                                   # both ends (partial work items) and a random interior
    mid = torch.randint(k, rows - k, (k,), generator=gen, device=DEV)
    return torch.cat((torch.arange(k, device=DEV), mid, torch.arange(rows - k, rows, device=DEV))).unique()


def _state_np(p, opt, sel):
    st = opt.state[p]
    pick = (lambda t: t.detach()) if sel is None else (lambda t: t.detach()[sel])
    return [pick(t).cpu().numpy().copy() for t in (p, p.grad, st["exp_avg"], st["exp_avg_sq"])]


def _run_schedule(p, opt, rows, gen, offset_grad=False):
    """Five steps through every mask kind, both eps values and bias corrections near 0.1 and near 1."""
    lr, betas = opt.param_groups[0]["lr"], opt.param_groups[0]["betas"]
    sel = _rows_to_compare(rows, p.numel() // rows, gen)
    schedule = [(1, "dense", 1e-8), (2, "random", 1e-15), (1000, "random", 1e-8), (1001, "none", 1e-15),
                (1002, "dense", 1e-15)]
    for t, kind, eps in schedule:
        opt.param_groups[0]["eps"] = eps
        g = torch.randn(p.numel() + 1, generator=gen, device=DEV)
        p.grad = (g[1:] if offset_grad else g[:-1]).view(p.shape)
        vis = None
        if kind == "random":
            vis = torch.rand(rows, generator=gen, device=DEV) < 0.3
        elif kind == "none":
            vis = torch.zeros(rows, dtype=torch.bool, device=DEV)
        if vis is not None:
            p.grad[~vis] = float("nan")                        # the gradient of a masked row is never read
        if opt.state[p]:
            opt.state[p]["step"].fill_(t - 1)
        else:
            assert t == 1
            opt.step(visibility=torch.zeros(rows, dtype=torch.bool, device=DEV))   # creates the state, moves nothing
            opt.state[p]["step"].fill_(0)
        before_full = [t_.detach().clone() for t_ in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])]
        before = _state_np(p, opt, sel)
        opt.step(visibility=vis)
        after_full = (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])
        if vis is not None:                                     # every masked row of the whole table, bitwise
            for b, a in zip(before_full, after_full):
                assert torch.equal(b[~vis].view(torch.int32), a[~vis].view(torch.int32))
        shown = torch.ones(rows, dtype=torch.bool, device=DEV) if vis is None else vis
        for a in after_full:
            assert bool(torch.isfinite(a[shown]).all())
        if bool(shown.any()):
            assert bool((after_full[0][shown] != before_full[0][shown]).any())
        after = _state_np(p, opt, sel)
        v_np = None if vis is None else (vis if sel is None else vis[sel]).cpu().numpy()
        assert_step_matches_oracle(before, (after[0], after[2], after[3]), t, lr, betas, eps, visible=v_np)


@pytest.mark.parametrize("rows", [1, 37, 100_003])
@pytest.mark.parametrize("row_len", [1, 3, 4, 45, 48, 64, 100, 256, 512, 513, 1024])
def test_steps_match_the_oracle(row_len, rows):
    gen = torch.Generator(device=DEV).manual_seed(row_len * 131 + rows)
    shape = (rows, 15, 3) if row_len == 45 else (rows, row_len)
    p = torch.nn.Parameter(torch.randn(shape, generator=gen, device=DEV))
    opt = GaussianAdam([{"params": [p], "row_sparse": True}], lr=1e-2)
    _run_schedule(p, opt, rows, gen)


@pytest.mark.parametrize("rows,row_len", [(37, 256), (1001, 48), (100_003, 4)])
def test_storage_offset_by_one_float_takes_the_scalar_path(rows, row_len):
    """param, grad and both moments start 4 bytes into their buffers: only 4-byte aligned."""
    gen = torch.Generator(device=DEV).manual_seed(7)
    n = rows * row_len
    p = torch.nn.Parameter(torch.randn(n + 1, generator=gen, device=DEV)[1:].view(rows, row_len))
    assert p.data_ptr() % 16 == 4 and p.is_contiguous()
    opt = GaussianAdam([{"params": [p], "row_sparse": True}], lr=1e-2)
    opt.state[p] = {"step": torch.tensor(0.0), "exp_avg": torch.zeros(n + 1, device=DEV)[1:].view(rows, row_len),
                    "exp_avg_sq": torch.zeros(n + 1, device=DEV)[1:].view(rows, row_len)}
    _run_schedule(p, opt, rows, gen, offset_grad=True)


SHAPES9 = [(1000, 3), (1000, 1, 3), (1000, 15, 3), (1000, 1), (1000, 4), (1000, 256), (512, 64), (512,), (77, 5)]


def _pair(shapes, seed=0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    a = [torch.nn.Parameter(torch.randn(s, generator=gen, device=DEV)) for s in shapes]
    b = [torch.nn.Parameter(t.detach().clone()) for t in a]
    return a, b, gen


def test_thirty_dense_steps_match_torch_adam():
    mine, ref, gen = _pair(SHAPES9)
    a = GaussianAdam([{"params": mine[:6], "row_sparse": True, "lr": 2e-2}, {"params": mine[6:]}], lr=1e-3, eps=1e-15)
    b = torch.optim.Adam([{"params": ref[:6], "lr": 2e-2}, {"params": ref[6:]}], lr=1e-3, eps=1e-15)
    for _ in range(30):
        for p, q in zip(mine, ref):
            p.grad = torch.randn(p.shape, generator=gen, device=DEV)
            q.grad = p.grad.clone()
        a.step(visibility=torch.ones(1000, dtype=torch.bool, device=DEV))
        b.step()
    for p, q in zip(mine, ref):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(a.state[p]["exp_avg_sq"], b.state[q]["exp_avg_sq"], rtol=1e-5, atol=1e-30)
        torch.testing.assert_close(a.state[p]["exp_avg"], b.state[q]["exp_avg"], rtol=1e-5, atol=1e-6)
        assert float(a.state[p]["step"]) == 30


def _adam_launches(opt):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        opt.step()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if "sgb_adam_" in e.key)


def test_eight_tensors_are_one_launch_and_nine_are_two():
    params, _, gen = _pair(SHAPES9)
    for p in params:
        p.grad = torch.randn(p.shape, generator=gen, device=DEV)
    eight, nine = GaussianAdam(params[:8]), GaussianAdam(params)
    eight.step(), nine.step()                                   # module load outside the trace
    torch.cuda.synchronize()
    assert _adam_launches(eight) == 1
    assert _adam_launches(nine) == 2


def test_step_never_synchronises():
    params, _, gen = _pair(SHAPES9)
    for p in params:
        p.grad = torch.randn(p.shape, generator=gen, device=DEV)
    opt = GaussianAdam([{"params": params[:6], "row_sparse": True}, {"params": params[6:]}])
    vis = torch.rand(1000, generator=gen, device=DEV) < 0.5
    opt.step(visibility=vis)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.step(visibility=vis)
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_two_runs_from_one_state_are_bitwise_equal():
    a, b, gen = _pair(SHAPES9[:6], seed=5)
    oa = GaussianAdam([{"params": a, "row_sparse": True}], lr=1e-2)
    ob = GaussianAdam([{"params": b, "row_sparse": True}], lr=1e-2)
    for _ in range(3):
        vis = torch.rand(1000, generator=gen, device=DEV) < 0.6
        for p, q in zip(a, b):
            p.grad = torch.randn(p.shape, generator=gen, device=DEV)
            q.grad = p.grad.clone()
        oa.step(visibility=vis), ob.step(visibility=vis)
    for p, q in zip(a, b):
        assert torch.equal(p, q) and torch.equal(oa.state[p]["exp_avg"], ob.state[q]["exp_avg"])
        assert torch.equal(oa.state[p]["exp_avg_sq"], ob.state[q]["exp_avg_sq"])


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


def _views(cams):
    return [SimpleNamespace(image_width=c.image_width, image_height=c.image_height, FoVx=c.FoVx, FoVy=c.FoVy,
                            world_view_transform=torch.as_tensor(c.world_view_transform, device=DEV),
                            full_proj_transform=torch.as_tensor(c.full_proj_transform, device=DEV),
                            camera_center=torch.as_tensor(c.camera_center, device=DEV)) for c in cams]


def test_short_rgb_fit_with_density_control_under_sparse_adam():
    """The loop of test_train_loop_gpu.py with optimizer_type="sparse_adam" and step(visibility=vis)."""
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.renderer import render
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    torch.manual_seed(0)
    scene = make_scene(4000, seed=21, sh=True, scale_mean=0.05)
    gt = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs, device=DEV)
    views = _views(orbit_cameras(6, 160, 120))
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        targets = [render(v, gt, Pipe, bg)["render"].clone() for v in views]
    rng = np.random.default_rng(0)
    keep = rng.choice(4000, 1500, replace=False)
    pts = scene.xyz[keep] + rng.normal(0, 0.01, (1500, 3)).astype(np.float32)
    m = GaussianModel(3).create_from_pcd(pts, rng.uniform(0.3, 0.7, (1500, 3)), spatial_lr_scale=1.0, device=DEV)
    m.active_sh_degree = 0
    args = SimpleNamespace(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                           position_lr_max_steps=300, feature_lr=2.5e-3, opacity_lr=0.05, scaling_lr=5e-3, rotation_lr=1e-3,
                           optimizer_type="sparse_adam")
    m.training_setup(args)
    assert type(m.optimizer) is GaussianAdam
    P0 = m._xyz.shape[0]
    losses, counts = [], []
    for it in range(1, 241):
        m.update_learning_rate(it)
        out = render(views[it % len(views)], m, Pipe, bg)
        loss = (out["render"] - targets[it % len(views)]).abs().mean()
        loss.backward()
        losses.append(float(loss))
        with torch.no_grad():
            vis, radii = out["visibility_filter"], out["radii"]
            m.max_radii2D[vis] = torch.max(m.max_radii2D[vis], radii[vis].float())
            m.add_densification_stats(out["viewspace_points"], vis)
            if it % 60 == 0:
                counts.append(m.densify_and_prune(0.0002, 0.005, 3.0, None))
                # density control renumbers the Gaussians: this view's mask no longer describes them
                vis = None
            m.optimizer.step(visibility=vis)
            m.optimizer.zero_grad(set_to_none=True)
    first, last = float(np.mean(losses[:10])), float(np.mean(losses[-10:]))
    assert np.isfinite(losses).all()
    assert last < 0.8 * first, (first, last)
    assert sum(c["cloned"] + c["split"] for c in counts) > 0
    assert m._xyz.shape[0] != P0 and m._xyz.shape[0] == m.max_radii2D.shape[0] == m.denom.shape[0]
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        assert p.shape[0] == m._xyz.shape[0]
        st = m.optimizer.state[p]
        assert st["exp_avg"].shape == p.shape and st["exp_avg_sq"].shape == p.shape
    m.reset_opacity()
    assert float(m.get_opacity.max()) <= 0.0100001
    out = render(views[0], m, Pipe, bg)
    (out["render"] - targets[0]).abs().mean().backward()
    m.optimizer.step(visibility=out["visibility_filter"])
    assert torch.isfinite(m._opacity).all() and m._opacity.grad is not None


@pytest.mark.parametrize("loss_type", ["cosine", "l2"])
def test_feature_fit_over_two_views_leaves_unseen_rows_alone(loss_type):
    """test_feature_loss_gpu.py's feature fit with GaussianAdam on the (P, 64) table, two views per step through
    render_chn_batch: the loss falls by the same margin, and rows no view saw keep their initial bits."""
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.renderer import render_chn_batch
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    from semantic_gaussians_b200.semantic import feature_map_loss_and_grad
    C = 64
    scene = make_scene(20000, seed=12, channels=C, scale_mean=0.03)
    xyz = scene.xyz.copy()
    xyz[-1000:, 2] += 50.0                                      # far above every camera: behind its near plane
    pc = GaussianModel.from_activated(xyz, scene.scales, scene.rotations, scene.opacity, device=DEV)
    pc.active_sh_degree = 0
    views = _views(orbit_cameras(3, 320, 240)[1:])
    feats0 = torch.as_tensor(scene.features, device=DEV)
    img_dim = [256, 192]
    bg = torch.zeros(C, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
        other = torch.randn(feats0.shape, generator=g, device=DEV)
        fmaps = [o["render"].half() for o in render_chn_batch(views, pc, Pipe, bg, num_channels=C, override_color=other,
                                                              override_shape=img_dim)]
    feats = feats0.clone().requires_grad_(True)
    opt = GaussianAdam([{"params": [feats], "lr": 0.05, "row_sparse": True}])
    seen = torch.zeros(feats.shape[0], dtype=torch.bool, device=DEV)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        outs = render_chn_batch(views, pc, Pipe, bg, num_channels=C, override_color=feats, override_shape=img_dim)
        pairs = [feature_map_loss_and_grad(o["render"], f, loss_type) for o, f in zip(outs, fmaps)]
        torch.autograd.backward([o["render"] for o in outs], [gr for _, gr in pairs])
        vis = visible_rows(outs)
        opt.step(visibility=vis)
        seen |= vis
        losses.append(sum(float(l) for l, _ in pairs))
    assert losses[-1] < 0.5 * losses[0], losses
    assert 1000 <= int((~seen).sum()) < feats.shape[0] // 2
    assert torch.equal(feats.detach()[~seen].view(torch.int32), feats0[~seen].view(torch.int32))
    assert not torch.equal(feats.detach()[seen], feats0[seen])
    st = opt.state[feats]
    assert float(st["exp_avg"][~seen].abs().max()) == 0.0 and float(st["exp_avg_sq"][~seen].abs().max()) == 0.0
