"""GPU: the 3D distillation sample and loss.  ElasticDistortion, the float64 Voxelizer and FeatureDataset[i] bitwise
against the reference's own objects (tests/golden/distill_golden.npz), voxel_indices on float64 against the numpy
oracle, voxel_feature_loss_and_grad against a float64 torch restatement of distill.py's three losses and their
autograd gradients, and one MinkUNet14A step against the torch-loss step."""
import os
import sys

import numpy as np
import pytest
import torch
from feature_loss_ref import feature_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_distill_golden import (DATASET_CASES, ELASTIC_CASES, ELASTIC_PARAMS, ROTATION_BOUND, SCALE_BOUND,  # noqa: E402
                                 VOX_CASES, VOXEL_SIZE, elastic_input, seed_all, vox_input, write_scene)
from make_raster_golden import digest  # noqa: E402

from oracle import voxel_oracle as vo  # noqa: E402
from semantic_gaussians_b200 import sparse as sp  # noqa: E402
from semantic_gaussians_b200.feature_dataset import ElasticDistortion, FeatureDataset, collate_fn  # noqa: E402
from semantic_gaussians_b200.mink_unet import mink_unet  # noqa: E402
from semantic_gaussians_b200.semantic import voxel_feature_loss_and_grad  # noqa: E402
from semantic_gaussians_b200.voxelize import Voxelizer, voxel_indices  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "distill_golden.npz"))
DEV = "cuda"


@pytest.mark.parametrize("as_tensor", [True, False])
@pytest.mark.parametrize("case", sorted(ELASTIC_CASES))
def test_elastic_distortion_is_reference_golden(case, as_tensor):
    xyz = elastic_input(case)
    inp = torch.from_numpy(xyz).to(DEV) if as_tensor else xyz
    seed_all(ELASTIC_CASES[case][0])
    got = ElasticDistortion(ELASTIC_PARAMS)(inp)
    if as_tensor:
        assert got.is_cuda
        got = got.cpu().numpy()
    skipped = len(GOLDEN[f"{case}_noise_dims"]) == 0
    assert got.dtype == (xyz.dtype if skipped else np.float64)
    assert np.array_equal(digest(got), GOLDEN[f"{case}_xyz.sha256"])


@pytest.mark.parametrize("as_tensor", [True, False])
def test_voxelizer_float64_is_reference_golden(as_tensor):
    case = "vox_f64"
    xyz, feats = vox_input(case)
    vox = Voxelizer(voxel_size=VOXEL_SIZE, use_augmentation=True, scale_augmentation_bound=SCALE_BOUND,
                    rotation_augmentation_bound=ROTATION_BOUND)
    seed_all(VOX_CASES[case][0])
    if as_tensor:
        coords, f, _, inverse, inds = vox.voxelize(torch.from_numpy(xyz).to(DEV), torch.from_numpy(feats).to(DEV),
                                                   None, return_ind=True)
        coords, f, inverse, inds = (t.cpu().numpy() for t in (coords, f, inverse, inds))
    else:
        coords, f, _, inverse, inds = vox.voxelize(xyz, feats, None, return_ind=True)
    assert np.array_equal(inds, GOLDEN[f"{case}_inds"]) and np.array_equal(inverse, GOLDEN[f"{case}_inverse"])
    assert np.array_equal(digest(coords), GOLDEN[f"{case}_coords.sha256"])
    assert np.array_equal(digest(f), GOLDEN[f"{case}_feats.sha256"])


@pytest.mark.parametrize("voxel_size", [0.02, 0.05])
def test_voxel_indices_float64_matches_oracle(voxel_size):
    rng = np.random.default_rng(7)
    xyz = rng.uniform(-3, 4, (30000, 3)) + rng.uniform(-1e-9, 1e-9, (30000, 3))
    xyz[:5000] = np.round(xyz[:5000] / voxel_size) * voxel_size     # points on voxel faces
    T = np.eye(4)[:3] / voxel_size
    first, inverse, coords = voxel_indices(torch.from_numpy(xyz).to(DEV), T)
    want_first, want_inverse, want_coords, _ = vo.voxelize(xyz, T)
    assert np.array_equal(first.cpu().numpy(), want_first)
    assert np.array_equal(inverse.cpu().numpy(), want_inverse)
    assert np.array_equal(coords.cpu().numpy(), want_coords)


@pytest.mark.parametrize("case", sorted(DATASET_CASES))
def test_feature_dataset_sample_is_reference_golden(case, tmp_path):
    seed, _, _, feature_type, aug = DATASET_CASES[case]
    gdir, pdir = write_scene(case, str(tmp_path))
    ds = FeatureDataset(gdir, pdir, 30000, VOXEL_SIZE, aug, feature_type)
    assert len(ds) == 1
    seed_all(seed)
    sample = ds[0]
    assert sample[4] == 0
    for name, t in zip(("locs", "features", "features_gt", "mask"), sample[:4]):
        assert t.is_cuda, name
        assert np.array_equal(digest(t.cpu().numpy()), GOLDEN[f"{case}_{name}.sha256"]), name


# ---------------------------------------------------------------- loss

def _loss_inputs(M, F, C, dtype, seed=0, p=0.6, zero_rows=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    output = torch.randn(M, F, device=DEV, generator=g)
    mask = torch.rand(M, device=DEV, generator=g) < p
    gt = torch.randn(int(mask.sum()), C, device=DEV, generator=g)
    if zero_rows:
        gt[::5] = 0
    return output, mask, gt.to(dtype)


def _reference(output, mask, gt, loss_type, head, C):
    """feature_loss_ref.feature_loss on the head's columns of the masked rows: (loss, count, d loss / d output)."""
    cols = slice(head * C, (head + 1) * C)
    loss, count, g = feature_loss(output[mask][:, cols], gt, loss_type)
    grad = torch.zeros_like(output, dtype=torch.float64)
    grad[mask, cols] = g
    return loss, count, grad


def _check(output, mask, gt, loss_type, head, C):
    loss, count, grad = voxel_feature_loss_and_grad(output, mask, gt, loss_type, head=head, channels=C)
    assert loss.dtype == count.dtype == torch.float64 and loss.ndim == count.ndim == 0
    assert grad.shape == output.shape and grad.dtype == torch.float32
    want_loss, want_count, want_grad = _reference(output, mask, gt, loss_type, head, C)
    assert count.item() == want_count
    assert abs(loss.item() - want_loss) <= 1e-5 * abs(want_loss) + 1e-12, (loss.item(), want_loss)
    err = (grad.double() - want_grad).abs().max().item()
    scale = want_grad.abs().max().item()
    assert err <= 1e-5 * scale + 1e-30, (err, scale)
    outside = torch.ones_like(grad, dtype=torch.bool)
    outside[:, head * C:(head + 1) * C] = ~mask[:, None]
    assert not grad[outside].any()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("loss_type", ["cosine", "l1", "l2"])
@pytest.mark.parametrize("F,C,head", [(1536, 768, 0), (1536, 768, 1), (5, 5, 0), (17, 5, 2), (768, 768, 0)])
def test_voxel_loss_matches_float64_restatement(F, C, head, loss_type, dtype):
    output, mask, gt = _loss_inputs(3001, F, C, dtype)
    _check(output, mask, gt, loss_type, head, C)


@pytest.mark.parametrize("loss_type", ["cosine", "l1", "l2"])
def test_voxel_loss_empty_mask_and_zero_targets(loss_type):
    output, mask, gt = _loss_inputs(1000, 1536, 768, torch.float16, p=0.0)
    assert gt.shape[0] == 0
    loss, count, grad = voxel_feature_loss_and_grad(output, mask, gt, loss_type, head=1)
    assert loss.item() == 0 and count.item() == 0 and not grad.any()
    output, mask, gt = _loss_inputs(1000, 1536, 768, torch.float32, seed=1)
    gt.zero_()
    if loss_type == "cosine":      # no row to average over: the reference skips the batch
        loss, count, grad = voxel_feature_loss_and_grad(output, mask, gt, loss_type, head=1)
        assert loss.item() == 0 and count.item() == 0 and not grad.any()
    else:
        _check(output, mask, gt, loss_type, 1, 768)


def test_voxel_loss_row_count_mismatch_is_nan():
    output, mask, gt = _loss_inputs(1000, 768, 768, torch.float16)
    loss, count, _ = voxel_feature_loss_and_grad(output, mask, gt[:-1], "l1")
    assert torch.isnan(loss) and torch.isnan(count)


@pytest.mark.parametrize("loss_type", ["cosine", "l1", "l2"])
def test_voxel_loss_two_calls_are_bitwise_equal(loss_type):
    output, mask, gt = _loss_inputs(50000, 1536, 768, torch.float16, seed=3)
    a = voxel_feature_loss_and_grad(output, mask, gt, loss_type, head=1)
    b = voxel_feature_loss_and_grad(output, mask, gt, loss_type, head=1)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("loss_type", ["cosine", "l1", "l2"])
def test_minkunet_step_matches_torch_loss(loss_type, tmp_path):
    """distill.py's step on a batch-2 collate of augmented samples: the fused loss's gradient fed to out.F.backward
    gives the parameter gradients of the torch loss's loss.backward()."""
    gdir, pdir = write_scene("ds_all", str(tmp_path))
    ds = FeatureDataset(gdir, pdir, 30000, VOXEL_SIZE, True, "all")
    batch = []
    for s in (1, 2):
        seed_all(s)
        batch.append(ds[0])
    locs, features, features_gt, mask, head_id = collate_fn(batch)
    assert locs[:, 0].unique().tolist() == [0, 1]
    C = features_gt.shape[1]
    torch.manual_seed(0)
    model = mink_unet(56, C, arch="MinkUNet14A").to(DEV)
    grads = []
    for fused in (True, False):
        model.zero_grad()
        out = model(sp.SparseTensor(features, locs))
        if fused:
            loss, count, grad = voxel_feature_loss_and_grad(out.F, mask, features_gt, loss_type, head_id, C)
            out.F.backward(grad)
        else:
            output = out.F[mask]
            y = features_gt.float()
            if loss_type == "cosine":
                nm = y.norm(dim=-1) > 0
                loss = (1 - torch.nn.CosineSimilarity()(output[nm][:, head_id * C:(head_id + 1) * C], y[nm])).mean()
            else:
                loss = (torch.nn.L1Loss() if loss_type == "l1" else torch.nn.MSELoss())(
                    output[:, head_id * C:(head_id + 1) * C], y)
            loss.backward()
        grads.append((loss.item(), {n: p.grad.double().clone() for n, p in model.named_parameters()}))
    (l_fused, g_fused), (l_torch, g_torch) = grads
    assert abs(l_fused - l_torch) <= 1e-5 * abs(l_torch)
    for n, g in g_torch.items():
        err = (g_fused[n] - g).norm().item()
        assert err <= 1e-5 * g.norm().item() + 1e-12, (n, err, g.norm().item())
