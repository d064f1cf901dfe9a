"""GPU: ConfusionMatrix (sgb_confusion_accumulate) against a numpy bincount restatement bit for bit, against the
reference's summed matrices (tests/golden/metric_golden.npz), and inside the reference's evaluation loop."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_metric_golden import CASES, metric_inputs  # noqa: E402
from metric_ref import confusion_full, reference_confusion  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NP_DTYPE = {torch.uint8: np.uint8, torch.int32: np.int32, torch.int64: np.int64}


def _labels(num_classes, n, pattern, pred_offset, rng):
    """(pred, gt) int64 numpy labels that the reference accepts: pred + pred_offset in [0, num_classes], gt in
    [0, num_classes], plus gt = num_classes + 1 (the wrap case) where the flat bin still fits."""
    hi = num_classes + 1 - pred_offset
    if pattern == "random":
        pred = rng.integers(0, hi, n)
        gt = rng.integers(0, num_classes + 1, n)
    else:   # long constant runs: whole warps hit one bin
        runs = max(1, n // 997 + 1)
        pred = np.repeat(rng.integers(0, hi, runs), 997)[:n]
        gt = np.repeat(rng.integers(0, num_classes + 1, runs), 997)[:n]
    wrap = (rng.random(n) < 0.03) & (pred + pred_offset < num_classes)
    gt = np.where(wrap, num_classes + 1, gt)
    return pred.astype(np.int64), gt.astype(np.int64)


def _check(cm, want_full):
    got = cm.matrix()
    assert got.dtype == np.uint64 and got.shape == (cm.num_classes + 1, cm.num_classes)
    assert np.array_equal(got, want_full[:, 1:])
    assert np.array_equal(cm.counts.cpu().numpy().astype(np.uint64), want_full)


@pytest.mark.parametrize("num_classes", [1, 19, 20, 200])
@pytest.mark.parametrize("pred_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("gt_dtype", [torch.uint8, torch.int32, torch.int64])
def test_matches_bincount(num_classes, pred_dtype, gt_dtype):
    from semantic_gaussians_b200.metric import ConfusionMatrix
    rng = np.random.default_rng(num_classes * 7 + pred_dtype.itemsize + gt_dtype.itemsize)
    for pattern in ("random", "constant"):
        for pred_offset in (0, 1):
            for n in (1, 3, 4099, 313_633):            # ragged N: the vector path's tail
                pred, gt = _labels(num_classes, n, pattern, pred_offset, rng)
                cm = ConfusionMatrix(num_classes, DEV)
                cm.add(torch.from_numpy(pred).to(DEV, pred_dtype), torch.from_numpy(gt).to(DEV, gt_dtype), pred_offset)
                want, invalid = confusion_full(pred, gt, num_classes, pred_offset)
                assert invalid == 0
                _check(cm, want)


@pytest.mark.parametrize("gt_dtype", [torch.uint8, torch.int32, torch.int64])
def test_unaligned_and_strided_views(gt_dtype):
    from semantic_gaussians_b200.metric import ConfusionMatrix
    rng = np.random.default_rng(5)
    nc, n = 20, 50_001
    pred, gt = _labels(nc, n + 8, "random", 1, rng)
    gt = np.minimum(gt, nc)           # the views below pair shifted elements: no wrap labels, every pair is legal
    P = torch.from_numpy(pred).to(DEV, torch.int32)
    G = torch.from_numpy(gt).to(DEV, gt_dtype)
    for a, b in ((1, 0), (0, 3), (2, 5), (3, 1)):        # element offsets: views off the 16-byte path
        cm = ConfusionMatrix(nc, DEV)
        cm.add(P[a:a + n], G[b:b + n], pred_offset=1)
        _check(cm, confusion_full(pred[a:a + n], gt[b:b + n], nc, 1)[0])
    cm = ConfusionMatrix(nc, DEV)                          # non-contiguous (H, W) views, every other column
    p2, g2 = P[: 100 * 400].view(100, 400)[:, ::2], G[: 100 * 400].view(100, 400)[:, 1::2]
    cm.add(p2, g2, pred_offset=1)
    _check(cm, confusion_full(p2.cpu().numpy(), g2.cpu().numpy(), nc, 1)[0])


def test_stack_of_views_over_many_ctas():
    from semantic_gaussians_b200.metric import ConfusionMatrix
    rng = np.random.default_rng(9)
    nc, V, H, W = 19, 8, 484, 648
    pred, gt = _labels(nc, V * H * W, "constant", 1, rng)
    cm = ConfusionMatrix(nc, DEV)
    cm.add(torch.from_numpy(pred).to(DEV).view(V, H, W), torch.from_numpy(gt).to(DEV, torch.uint8).view(V, H, W), 1)
    _check(cm, confusion_full(pred, gt, nc, 1)[0])


@pytest.mark.parametrize("case", sorted(CASES))
def test_matches_reference_golden(case):
    from semantic_gaussians_b200.metric import ConfusionMatrix, confusion_matrix
    nc = CASES[case][0]
    golden = np.load(os.path.join(ROOT, "tests", "golden", "metric_golden.npz"))[f"{case}_matrix"]
    cm = ConfusionMatrix(nc, DEV)
    total = np.zeros_like(golden)
    for i, (pred, gt) in enumerate(metric_inputs(case)):
        p, g = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
        cm.add(p, g.to(torch.uint8) if i % 2 else g, pred_offset=1)
        total += confusion_matrix(p + 1, g, nc)               # one-shot drop-in of the reference function
    assert np.array_equal(cm.matrix(), golden)
    assert np.array_equal(total, golden)


def test_adds_on_two_streams_then_one_read():
    from semantic_gaussians_b200.metric import ConfusionMatrix
    rng = np.random.default_rng(3)
    nc = 20
    cm = ConfusionMatrix(nc, DEV)
    inputs = [_labels(nc, n, pat, 1, rng) for n, pat in ((100_003, "random"), (70_001, "constant"),
                                                         (4097, "random"), (250_000, "constant"))]
    dev_inputs = [(torch.from_numpy(p).to(DEV), torch.from_numpy(g).to(DEV, torch.int32)) for p, g in inputs]
    streams = [torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream(DEV))         # inputs and the zeroed counts are ready
    for i, (p, g) in enumerate(dev_inputs):
        with torch.cuda.stream(streams[i % 2]):
            cm.add(p, g, pred_offset=1)
    want = sum(confusion_full(p, g, nc, 1)[0] for p, g in inputs)
    _check(cm, want)


@pytest.mark.parametrize("pred,gt,pred_offset,ref_raises", [
    ([3, -1, 2], [1, 2, 3], 0, True),               # negative prediction
    ([3, 1, 2], [1, -2, 3], 0, False),              # negative ground truth (numpy folds 1 * 20 - 2 into row 0)
    ([0, 1, 19], [1, 2, 3], 1, True),               # pred + offset == nb: the flat bin is past the end
    ([19, 1, 2], [20, 2, 3], 0, True),              # last row, gt = num_classes + 1: flat bin == nb * nb
    ([0, 1, 2], [1, 2, 401], 0, True),              # ground truth past the end from row 2
    ([0, 1, 2], [1, 2, 10 ** 12], 0, False),        # far past the end (numpy would allocate 10^12 bins first)
    ([2 ** 63 - 1, 1, 2], [1, 2, 3], 1, False),     # pred + offset past int64 (numpy wraps it into bin 1)
    ([-1, 1, 2], [1, 2, 3], 1, False),              # -1 + 1 = 0 is legal: the control case
])
def test_out_of_range_pairs_raise_until_reset(pred, gt, pred_offset, ref_raises):
    from semantic_gaussians_b200.metric import ConfusionMatrix
    nc = 19
    p = torch.tensor(pred, dtype=torch.int64, device=DEV)
    g = torch.tensor(gt, dtype=torch.int64, device=DEV)
    want, invalid = confusion_full(np.array(pred), np.array(gt), nc, pred_offset)
    cm = ConfusionMatrix(nc, DEV)
    cm.add(p, g, pred_offset)
    if invalid == 0:
        _check(cm, want)
        return
    with pytest.raises(ValueError, match="outside the confusion matrix"):
        cm.matrix()
    if ref_raises:                                            # the reference raises on the same view
        with pytest.raises(ValueError):
            reference_confusion(np.array(pred) + pred_offset, np.array(gt), nc)
    with pytest.raises(ValueError):                          # the count stays until reset()
        cm.matrix()
    cm.reset()
    assert np.array_equal(cm.matrix(), np.zeros((nc + 1, nc), np.uint64))
    ok = torch.tensor([0, 1, 2], dtype=torch.int64, device=DEV)
    cm.add(ok, ok, pred_offset=1)
    _check(cm, confusion_full(np.array([0, 1, 2]), np.array([0, 1, 2]), nc, 1)[0])


def test_argument_checks():
    from semantic_gaussians_b200 import _lib
    from semantic_gaussians_b200.metric import ConfusionMatrix
    cm = ConfusionMatrix(19, DEV)
    p = torch.zeros(10, dtype=torch.int64, device=DEV)
    with pytest.raises(ValueError):
        cm.add(p.cpu(), p)
    with pytest.raises(ValueError):
        cm.add(p, p[:9])
    with pytest.raises(ValueError):
        cm.add(p.float(), p)
    with pytest.raises(ValueError):
        cm.add(p.to(torch.uint8), p)                         # predictions are int32 / int64
    with pytest.raises(ValueError):
        cm.add(p, p.to(torch.int16))
    with pytest.raises(_lib.SgbError, match="num_classes = 226"):
        ConfusionMatrix(226, DEV)
    cm.add(p[:0], p[:0])
    assert cm.matrix().sum() == 0


class _Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


def test_reference_eval_loop_on_rendered_views():
    """eval_segmentation.py's per-view loop (pred_on_3d and feature-image modes) on this repository's renderer:
    the reference's .cpu() + numpy confusion equals what ConfusionMatrix accumulates from the same renders with no
    synchronisation between views."""
    from types import SimpleNamespace

    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.metric import ConfusionMatrix
    from semantic_gaussians_b200.renderer import render_chn
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    from semantic_gaussians_b200.semantic import label_argmax

    Cf, K = 32, 20                                            # feature width; 19 classes + "other"
    nc = K - 1
    scene = make_scene(30000, seed=4, channels=Cf)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=DEV)
    pc.active_sh_degree = 0
    features = torch.as_tensor(scene.features, device=DEV).contiguous()
    g = torch.Generator(device=DEV).manual_seed(0)
    text_features = torch.nn.functional.normalize(torch.randn(K, Cf, generator=g, device=DEV), dim=1)
    views = [SimpleNamespace(image_width=c.image_width, image_height=c.image_height, FoVx=c.FoVx, FoVy=c.FoVy,
                             world_view_transform=torch.as_tensor(c.world_view_transform, device=DEV),
                             full_proj_transform=torch.as_tensor(c.full_proj_transform, device=DEV),
                             camera_center=torch.as_tensor(c.camera_center, device=DEV))
             for c in orbit_cameras(5, 200, 150)]
    rng = np.random.default_rng(1)
    gts = [rng.integers(0, nc + 1, (150, 200)).astype(np.uint8) for _ in views]

    with torch.no_grad():
        sim = torch.einsum("cq,dq->dc", text_features, features)
        label_soft = sim.softmax(dim=1)
        bg_k, bg_c = torch.zeros(K, device=DEV), torch.zeros(Cf, device=DEV)
        for mode in ("pred_on_3d", "feature_image"):
            renders, labels = [], []
            cm = ConfusionMatrix(nc, DEV)
            for view, gt in zip(views, gts):
                if mode == "pred_on_3d":
                    rendering = render_chn(view, pc, _Pipe, bg_k, num_channels=K, override_color=label_soft)["render"]
                    label = label_argmax(rendering)                              # rendering[1:].argmax(dim=0)
                else:
                    rendering = render_chn(view, pc, _Pipe, bg_c, num_channels=Cf, override_color=features)["render"]
                    rendering = rendering / (rendering.norm(dim=0, keepdim=True) + 1e-8)
                    label = torch.einsum("cq,qhw->chw", text_features, rendering)[1:].argmax(dim=0)
                renders.append(rendering)
                labels.append(label)
                gt_dev = torch.from_numpy(gt).to(DEV, non_blocking=False)
                torch.cuda.set_sync_debug_mode("error")                      # add() must not synchronise
                try:
                    cm.add(label, gt_dev, pred_offset=1)
                finally:
                    torch.cuda.set_sync_debug_mode("default")
            got = cm.matrix()

            confusion = np.zeros((nc + 1, nc), dtype=np.ulonglong)            # the reference's statements
            for rendering, gt in zip(renders, gts):
                if mode == "pred_on_3d":
                    label = rendering[1:].argmax(dim=0).cpu()
                else:
                    label = torch.einsum("cq,qhw->chw", text_features, rendering)[1:].argmax(dim=0).cpu()
                label += 1
                label_img = torch.from_numpy(gt).int().cpu()
                confusion += reference_confusion(label.cpu().numpy().reshape(-1), label_img.cpu().numpy().reshape(-1),
                                                 nc)
            assert confusion.sum() == len(views) * 150 * 200 - sum(int((g == 0).sum()) for g in gts)
            assert np.array_equal(got, confusion), mode
