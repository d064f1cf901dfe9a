"""Forward + backward time of the RGB training loss (train.py:141-149, lambda_dssim = 0.2):

  (a) torch   the reference's torch expressions (utils/loss_utils.py: five depthwise conv2d + elementwise ops),
              restated in tests/loss_ref.py, through autograd, with torch's default settings
  (b) fused   semantic_gaussians_b200.loss_utils.photometric_loss (csrc/loss.cu: one kernel each way)

at 3x1080x1920 and at 3x968x1296 with cut_edge, timed with CUDA events (warm-up, then --reps repetitions),
the two alternating --rounds times in one run.  Then one K2-size training step (1M Gaussians, 1080p:
render + loss + backward) with each loss, alternating the same way.

The achieved rate of (b) is stated against the algorithmic bytes, a floor computed from shapes (not measured):
44 B per plane-pixel (x, y in and a, b, c out forward; a, b, c, x, y in and the gradient out backward)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from loss_ref import photometric_torch, window  # noqa: E402
from semantic_gaussians_b200.loss_utils import photometric_loss  # noqa: E402

BYTES_PER_PLANE_PIXEL = 44


def loss_fns(dev):
    w32 = window(torch.float32, dev)
    return {"torch": lambda a, b, cut: photometric_torch(a, b, w32, 0.2, cut)[0],
            "fused": lambda a, b, cut: photometric_loss(a, b, 0.2, cut)[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--step-reps", type=int, default=20)
    ap.add_argument("--no-step", action="store_true", help="skip the K2-size training step")
    ap.add_argument("--profile", action="store_true", help="also report the two kernels' time (torch.profiler)")
    args = ap.parse_args()
    dev, gpu_name = gpu("time_loss.py")
    fns = loss_fns(dev)
    result = {"card": gpu_name, "loss": {}, "step": {}}

    g = torch.Generator(device=dev).manual_seed(0)
    for (C, H, W), cut in (((3, 1080, 1920), False), ((3, 968, 1296), True)):
        x = torch.rand((C, H, W), generator=g, device=dev).requires_grad_(True)
        y = torch.rand((C, H, W), generator=g, device=dev)
        h, w = (H - 2 * (H // 100), W - 2 * (W // 100)) if cut else (H, W)
        nbytes = BYTES_PER_PLANE_PIXEL * C * h * w

        def run(name):
            x.grad = None
            fns[name](x, y, cut).backward()

        key = f"{C}x{H}x{W}" + (" cut_edge" if cut else "")
        times = {"torch": [], "fused": []}
        for _ in range(args.rounds):
            for name in ("torch", "fused"):
                times[name].append(time_ms(lambda: run(name), args.reps, args.warmup))
        t_t, t_f = min(times["torch"]), min(times["fused"])
        print(f"{key}: torch fwd+bwd {', '.join(f'{t:.3f}' for t in times['torch'])} ms | "
              f"fused {', '.join(f'{t:.3f}' for t in times['fused'])} ms | best-of speed-up {t_t / t_f:.2f}x | "
              f"fused {nbytes / (t_f * 1e-3) / 1e9:.0f} GB/s against {nbytes / 1e9:.3f} GB algorithmic", flush=True)
        result["loss"][key] = {"torch_ms": times["torch"], "fused_ms": times["fused"],
                               "algorithmic_GB": nbytes / 1e9, "fused_GBps_best": nbytes / (t_f * 1e-3) / 1e9}
        if args.profile:
            k = kernel_ms(lambda: run("fused"), 20, ("ssim_fwd_kernel", "ssim_bwd_kernel"))
            tk = sum(k.values())
            print(f"{key}: kernels " + ", ".join(f"{n_} {v:.3f} ms" for n_, v in sorted(k.items())) +
                  f" | {nbytes / (tk * 1e-3) / 1e9:.0f} GB/s against the algorithmic bytes", flush=True)
            result["loss"][key]["kernel_ms"] = k
        del x, y

    if not args.no_step:
        from semantic_gaussians_b200.gaussian_model import GaussianModel
        from semantic_gaussians_b200.renderer import render
        from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras

        scene = make_scene(1_000_000, 0, sh=True)
        m = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs,
                                         device=dev)
        params = [m._xyz, m._opacity, m._scaling, m._rotation, m._features_dc, m._features_rest]
        for p in params:
            p.requires_grad_(True)
        views = device_views(orbit_cameras(8, 1920, 1080), dev)
        bg = torch.zeros(3, device=dev)
        gt = torch.rand((3, 1080, 1920), generator=g, device=dev)
        it = [0]

        def step(name):
            for p in params:
                p.grad = None
            v = views[it[0] % len(views)]
            it[0] += 1
            out = render(v, m, Pipe, bg)
            fns[name](out["render"], gt, False).backward()

        times = {"torch": [], "fused": []}
        for _ in range(args.rounds):
            for name in ("torch", "fused"):
                times[name].append(time_ms(lambda: step(name), args.step_reps, 3))
        print(f"K2 step (1M Gaussians, 1080p, render + loss + backward): torch loss "
              f"{', '.join(f'{t:.2f}' for t in times['torch'])} ms | fused loss "
              f"{', '.join(f'{t:.2f}' for t in times['fused'])} ms", flush=True)
        result["step"]["k2_1080p"] = times
    print(json.dumps(result))


if __name__ == "__main__":
    main()
