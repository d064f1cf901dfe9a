"""GPU: semantic.voxel_feature_loss, the 3D distillation loss as an autograd function of an fp32 / fp16 / bf16 network
output.  On fp32 output its loss, count and gradient are bitwise voxel_feature_loss_and_grad's; on half output they are
that call's on the upcast output, with the upstream scale applied before the one rounding to the half type.  The
unscaled half gradient is checked against the float64 restatement at distillation size, a MinkUNet14A step under fp16
autocast with GradScaler and under bf16, and the call runs without a host sync, within the half gradient's memory and
reproducibly."""
import os
import sys

import pytest
import torch
from feature_loss_ref import feature_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_distill_golden import VOXEL_SIZE, seed_all, write_scene  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200 import sparse as sp  # noqa: E402
from semantic_gaussians_b200.feature_dataset import FeatureDataset, collate_fn  # noqa: E402
from semantic_gaussians_b200.mink_unet import mink_unet  # noqa: E402
from semantic_gaussians_b200.semantic import voxel_feature_loss, voxel_feature_loss_and_grad  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
LOSSES = ["cosine", "l1", "l2"]
BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}


def _inputs(M, F, C, out_dtype, gt_dtype, seed=0, p=0.6):
    """(M, F) output in out_dtype, a p-masked row mask and one (C) target row per masked row, every fifth one zero."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    output = torch.randn(M, F, device=DEV, generator=g).to(out_dtype)
    mask = torch.rand(M, device=DEV, generator=g) < p
    gt = torch.randn(int(mask.sum()), C, device=DEV, generator=g)
    gt[::5] = 0
    return output, mask, gt.to(gt_dtype)


def _bitwise_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(BITS[a.dtype]), b.view(BITS[b.dtype]))


def _same_scalar(a, b):
    return (torch.isnan(a) and torch.isnan(b)) or torch.equal(a, b)


def _check_against_fused(output, mask, gt, loss_type, head, C, scale=1.0):
    """voxel_feature_loss on output, then (scale * loss).backward(), against voxel_feature_loss_and_grad on
    output.float(): the same loss and count, and output.grad == (g_ref * scale).to(output.dtype), bit for bit."""
    want_loss, want_count, g_ref = voxel_feature_loss_and_grad(output.float(), mask, gt, loss_type, head=head,
                                                               channels=C)
    x = output.detach().clone().requires_grad_(True)
    loss, count = voxel_feature_loss(x, mask, gt, loss_type, head=head, channels=C)
    assert loss.dtype == count.dtype == torch.float64 and loss.ndim == count.ndim == 0
    assert loss.requires_grad and not count.requires_grad
    assert _same_scalar(loss.detach(), want_loss) and _same_scalar(count, want_count)
    (scale * loss).backward()
    assert x.grad.dtype == output.dtype
    assert _bitwise_equal(x.grad, (g_ref * scale).to(output.dtype))


# ---------------------------------------------------------------- bitwise relations

SHAPES = [(2, 1, 1), (31, 31, 0), (64, 31, 1), (1536, 768, 0), (1536, 768, 1), (1024, 1024, 0), (2048, 1024, 1)]


@pytest.mark.parametrize("gt_dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("loss_type", LOSSES)
@pytest.mark.parametrize("F,C,head", SHAPES)
def test_fp32_output_is_the_fused_call(F, C, head, loss_type, gt_dtype):
    output, mask, gt = _inputs(3001, F, C, torch.float32, gt_dtype)
    _check_against_fused(output, mask, gt, loss_type, head, C)


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("loss_type", LOSSES)
def test_edge_cases_are_the_fused_call(loss_type, out_dtype):
    # every target row zero: the cosine count is 0 (loss and gradient 0); l1 / l2 average as usual
    output, mask, gt = _inputs(1000, 1536, 768, out_dtype, torch.float32, seed=1)
    _check_against_fused(output, mask, gt.zero_(), loss_type, 1, 768)
    # an empty mask, and M = 0
    output, mask, gt = _inputs(1000, 1536, 768, out_dtype, torch.float16, p=0.0)
    assert gt.shape[0] == 0
    _check_against_fused(output, mask, gt, loss_type, 1, 768)
    _check_against_fused(output[:0], mask[:0], gt, loss_type, 1, 768)
    # the mask selects other than features_gt's row count: NaN loss and count
    output, mask, gt = _inputs(1000, 768, 768, out_dtype, torch.float16, seed=2)
    x = output.detach().clone().requires_grad_(True)
    loss, count = voxel_feature_loss(x, mask, gt[:-1], loss_type)
    assert torch.isnan(loss) and torch.isnan(count)
    _check_against_fused(output, mask, gt[:-1], loss_type, 0, 768)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 16])
@pytest.mark.parametrize("gt_dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("loss_type", LOSSES)
@pytest.mark.parametrize("F,C,head", [(31, 31, 0), (1536, 768, 1), (2048, 1024, 1)])
def test_half_output_is_the_fused_call_on_the_upcast(F, C, head, loss_type, out_dtype, gt_dtype, scale):
    output, mask, gt = _inputs(3001, F, C, out_dtype, gt_dtype, seed=4)
    _check_against_fused(output, mask, gt, loss_type, head, C, scale)


# ---------------------------------------------------------------- float64

@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("loss_type", LOSSES)
def test_half_gradient_against_float64_at_distillation_size(loss_type, out_dtype):
    """1 M rows x 768, 60 % masked: on the rounded inputs the unscaled gradient is within fp32 accumulation error
    (1e-5 of the largest gradient element, as for the fp32 call) plus one rounding to the half type: u |ref| for a
    normal result (u = 2^-11 fp16, 2^-8 bf16), half the smallest subnormal below the normal range."""
    output, mask, gt = _inputs(1_000_000, 768, 768, out_dtype, torch.float16, seed=5)
    x = output.detach().clone().requires_grad_(True)
    loss, count = voxel_feature_loss(x, mask, gt, loss_type)
    loss.backward()
    want_loss, want_count, want = feature_loss(output[mask], gt, loss_type)
    assert count.item() == want_count
    assert abs(loss.item() - want_loss) <= 1e-5 * abs(want_loss) + 1e-12, (loss.item(), want_loss)
    got = x.grad[mask].double()
    assert not x.grad[~mask].any()
    del x, output
    fi = torch.finfo(out_dtype)
    u, half_tiny = fi.eps / 2, fi.smallest_normal * fi.eps / 2
    bound = 1e-5 * want.abs().max() + u * want.abs() + half_tiny
    excess = ((got - want).abs() - bound).max().item()
    assert excess <= 0, (excess, want.abs().max().item())


# ---------------------------------------------------------------- a MinkUNet14A step

def _sample(tmp_path):
    gdir, pdir = write_scene("ds_all", str(tmp_path))
    ds = FeatureDataset(gdir, pdir, 30000, VOXEL_SIZE, True, "all")
    seed_all(1)
    return collate_fn([ds[0]])


@pytest.mark.parametrize("loss_type", LOSSES)
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16])
def test_minkunet_step_under_autocast(out_dtype, loss_type, tmp_path):
    """fp16 with GradScaler: the gradient reaching out.F is the .float() route's gradient times the scale, rounded
    once, and the scaler steps (no inf found).  bf16 without a scaler: the .float() route's gradient, rounded once."""
    locs, features, features_gt, mask, head_id = _sample(tmp_path)
    C = features_gt.shape[1]
    torch.manual_seed(0)
    model = mink_unet(56, C, arch="MinkUNet14A").to(DEV)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda") if out_dtype == torch.float16 else None
    with torch.autocast("cuda", dtype=out_dtype):
        out = model(sp.SparseTensor(features, locs))
    assert out.F.dtype == out_dtype
    out.F.retain_grad()
    _, _, g_ref = voxel_feature_loss_and_grad(out.F.detach().float(), mask, features_gt, loss_type, head_id, C)
    loss, count = voxel_feature_loss(out.F, mask, features_gt, loss_type, head_id, C)
    assert count.item() > 0
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    opt.zero_grad()
    if scaler is not None:
        scale = scaler.get_scale()
        scaler.scale(loss).backward()
        assert _bitwise_equal(out.F.grad, (g_ref * scale).to(out_dtype))
        assert (out.F.grad != 0).sum() > 0.9 * (g_ref != 0).sum()
        scaler.step(opt)
        scaler.update()
        assert scaler.get_scale() == scale          # an inf would have skipped the step and halved the scale
    else:
        loss.backward()
        assert _bitwise_equal(out.F.grad, g_ref.to(out_dtype))
        opt.step()
    moved = [n for n, p in model.named_parameters() if not torch.equal(p.detach(), before[n])]
    assert len(moved) > len(before) // 2, (len(moved), len(before))


# ---------------------------------------------------------------- sync, memory, determinism

@pytest.mark.parametrize("loss_type", LOSSES)
def test_no_sync_bounded_memory_and_reproducible(loss_type):
    M, F = 1_000_000, 768
    output, mask, gt = _inputs(M, F, 768, torch.bfloat16, torch.float16, seed=6)
    ws = _lib.load().sgb_voxel_feature_loss_workspace_bytes(M)
    runs = []
    for _ in range(2):
        x = output.detach().clone().requires_grad_(True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss, count = voxel_feature_loss(x, mask, gt, loss_type)
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        extra = torch.cuda.max_memory_allocated() - base
        assert extra <= M * F * 2 + ws + 2**20, (extra, M * F * 2, ws)
        runs.append((loss.detach(), count, x.grad))
    (l0, c0, g0), (l1, c1, g1) = runs
    assert torch.equal(l0, l1) and torch.equal(c0, c1) and _bitwise_equal(g0, g1)
