"""Per-view cost of the segmentation evaluation loop (eval_segmentation.py, default pred_on_3d mode) at the reference's
evaluation size: 1 M Gaussians (scene_synth.make_scene), 648x484 (config/eval.yaml), K = 20 rendered class
probabilities (19 ScanNet classes + "other"), 100 orbit views, ground truth generated from a seed.  The per-scene
softmax of the Gaussians' class similarities is computed once, outside both arms.  Per view:

  (a) reference   render_chn -> rendering[1:].argmax(dim=0).cpu() -> label += 1 ->
                  confusion += confusion_matrix(label.numpy(), gt (host int32), 19)   (numpy bincount, as utils/metric.py)
  (b) device      render_chn -> label_argmax -> ConfusionMatrix.add(label, gt, pred_offset=1), the uint8 ground truth
                  copied from pinned host memory without a sync; one matrix() read after the last view

The two arms alternate --rounds times in one process (host clock around each arm, which ends in a device sync); both
must give the identical matrix.  A separate torch.profiler pass reports the kernel time of sgb_confusion_accumulate."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from timing import Pipe, device_views, gpu  # noqa: E402

from metric_ref import reference_confusion  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.metric import ConfusionMatrix  # noqa: E402
from semantic_gaussians_b200.renderer import render_chn  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402
from semantic_gaussians_b200.semantic import feature_logits, label_argmax  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--width", type=int, default=648)
    ap.add_argument("--height", type=int, default=484)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--channels", type=int, default=64, help="width of the per-Gaussian features")
    args = ap.parse_args()
    dev, gpu_name = gpu("time_eval.py")
    K, nc, W, H = 20, 19, args.width, args.height

    scene = make_scene(args.gaussians, seed=0, channels=args.channels)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
    pc.active_sh_degree = 0
    features = torch.as_tensor(scene.features, device=dev).contiguous()
    g = torch.Generator(device=dev).manual_seed(0)
    text = torch.nn.functional.normalize(torch.randn(K, args.channels, generator=g, device=dev), dim=1)
    label_soft = feature_logits(features, text).softmax(dim=1)          # once per scene
    bg = torch.zeros(K, device=dev)
    views = device_views(orbit_cameras(args.views, W, H), dev)
    rng = np.random.default_rng(0)
    gts = [rng.integers(0, nc + 1, (H, W)).astype(np.uint8) for _ in views]     # 0 = unlabelled
    gts_pinned = [torch.from_numpy(x).pin_memory() for x in gts]

    def render(view):
        return render_chn(view, pc, Pipe, bg, num_channels=K, override_color=label_soft)["render"]

    def arm_reference(vs):
        confusion = np.zeros((nc + 1, nc), dtype=np.ulonglong)
        for view, gt in vs:
            label = render(view)[1:].argmax(dim=0).cpu()
            label += 1
            label_img = torch.from_numpy(gt).int().cpu()
            confusion += reference_confusion(label.numpy().reshape(-1), label_img.numpy().reshape(-1), nc)
        return confusion

    def arm_device(vs):
        cm = ConfusionMatrix(nc, dev)
        for view, gt in vs:
            cm.add(label_argmax(render(view)), gt.to(dev, non_blocking=True), pred_offset=1)
        return cm.matrix()

    with torch.no_grad():
        arm_reference(zip(views[:3], gts[:3]))                          # warm-up of every shape
        arm_device(zip(views[:3], gts_pinned[:3]))
        times = {"reference": [], "device": []}
        want = None
        for _ in range(args.rounds):
            for name, fn, gt_list in (("reference", arm_reference, gts), ("device", arm_device, gts_pinned)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                m = fn(zip(views, gt_list))
                times[name].append((time.perf_counter() - t0) * 1e3 / len(views))
                if want is None:
                    want = m
                if not np.array_equal(m, want):
                    raise SystemExit(f"{name}: confusion matrix differs from the first arm's")
        print(f"{len(views)} views, {args.gaussians} Gaussians, {W}x{H}, K = {K}: ms/view "
              f"reference (.cpu + numpy) {', '.join(f'{t:.3f}' for t in times['reference'])} | "
              f"device (ConfusionMatrix) {', '.join(f'{t:.3f}' for t in times['device'])} | "
              f"best-of {min(times['reference']) / min(times['device']):.2f}x", flush=True)
        print(f"matrices identical across arms and rounds: {int(want.sum())} labelled pixels counted", flush=True)
        print("confusion matrix (rows: prediction 0..19, columns: ground truth 1..19):", flush=True)
        print(want, flush=True)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            arm_device(zip(views, gts_pinned))
            torch.cuda.synchronize()
        k_ms, k_n = 0.0, 0
        for e in prof.key_averages():
            if "confusion_kernel" in e.key:
                k_ms += e.device_time_total / 1e3
                k_n += e.count
        print(f"sgb_confusion_accumulate kernel: {k_ms / max(k_n, 1) * 1e3:.2f} us per view "
              f"({k_n} launches, {W * H} pixels each)", flush=True)
    print(json.dumps({"card": gpu_name, "views": len(views), "ms_per_view": times,
                      "confusion_kernel_us_per_view": k_ms / max(k_n, 1) * 1e3, "kernel_launches": k_n}))


if __name__ == "__main__":
    main()
