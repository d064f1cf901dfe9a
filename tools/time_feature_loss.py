"""Time of the feature-map distillation loss and its gradient (distill.py:111-124):

  (a) torch   the reference's expressions applied per pixel of the rendered (C,H,W) image, the fp16 target cast to
              fp32, gradient through autograd:
                cosine  m = t.norm(dim=0) > 0;  (1 - F.cosine_similarity(render, t, dim=0))[m].mean()
                l1      F.l1_loss(render, t)          l2  F.mse_loss(render, t)
  (b) fused   semantic_gaussians_b200.semantic.feature_map_loss_and_grad (csrc/feature_loss.cu)

Both arms return (loss, d loss / d render).  Sizes: C = 256 at 1080x1920 (K3) and C = 512 at 968x1296 (K4), fp16
targets; the two arms alternate --rounds times per size, timed with CUDA events (warm-up, then --reps repetitions).
Then a K3-shaped step (1M Gaussians, 256 channels, 1080p: render_chn + cosine loss + backward) with each arm,
alternating the same way.  --profile adds a separate torch.profiler pass for the fused kernels' own time.

The achieved rate of (b) is stated against the algorithmic bytes computed from shapes (not measured): render read
once, target read once, gradient written once, N C (4 + 2 + 4) bytes with an fp16 target; the valid-pixel count of
the cosine loss reads on top of that the target up to each pixel's first non-zero channel (about one plane here)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.semantic import feature_map_loss_and_grad  # noqa: E402

KERNELS = ("count_valid_pixels_kernel", "feature_cosine_kernel", "feature_elementwise_kernel")


def torch_loss(render, target, loss_type):
    t = target.float()
    if loss_type == "cosine":
        m = t.norm(dim=0) > 0
        return (1 - F.cosine_similarity(render, t, dim=0))[m].mean()
    return F.l1_loss(render, t) if loss_type == "l1" else F.mse_loss(render, t)


def arms(loss_type):
    def torch_arm(render, target):
        loss = torch_loss(render, target, loss_type)
        return loss, torch.autograd.grad(loss, render)[0]

    def fused_arm(render, target):
        return feature_map_loss_and_grad(render, target, loss_type)

    return {"torch": torch_arm, "fused": fused_arm}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--step-reps", type=int, default=10)
    ap.add_argument("--no-step", action="store_true", help="skip the K3-shaped training step")
    ap.add_argument("--profile", action="store_true", help="also report the fused kernels' time (torch.profiler)")
    args = ap.parse_args()
    dev, gpu_name = gpu("time_feature_loss.py")
    result = {"card": gpu_name, "loss": {}, "step": {}}

    g = torch.Generator(device=dev).manual_seed(0)
    for C, H, W in ((256, 1080, 1920), (512, 968, 1296)):
        render = torch.randn((C, H, W), generator=g, device=dev).requires_grad_(True)
        target = (0.5 * render.detach() + torch.randn((C, H, W), generator=g, device=dev)).half()
        target[:, : H // 10] = 0                                    # some empty target pixels
        N = H * W
        nbytes = N * C * (4 + 2 + 4)
        for loss_type in ("cosine", "l1", "l2"):
            fns = arms(loss_type)
            key = f"{loss_type} {C}x{H}x{W} f16"
            lt, lf = fns["torch"](render, target)[0], fns["fused"](render, target)[0]
            times = {"torch": [], "fused": []}
            for _ in range(args.rounds):
                for name in ("torch", "fused"):
                    times[name].append(time_ms(lambda: fns[name](render, target), args.reps, args.warmup))
            t_t, t_f = min(times["torch"]), min(times["fused"])
            print(f"{key}: torch {', '.join(f'{t:.3f}' for t in times['torch'])} ms | "
                  f"fused {', '.join(f'{t:.3f}' for t in times['fused'])} ms | best-of speed-up {t_t / t_f:.2f}x | "
                  f"fused call {nbytes / (t_f * 1e-3) / 1e9:.0f} GB/s against {nbytes / 1e9:.3f} GB algorithmic | "
                  f"loss torch {float(lt.detach()):.9f} fused {float(lf):.9f}", flush=True)
            rec = {"torch_ms": times["torch"], "fused_ms": times["fused"], "algorithmic_GB": nbytes / 1e9,
                   "fused_call_GBps_best": nbytes / (t_f * 1e-3) / 1e9}
            if args.profile:
                k = kernel_ms(lambda: fns["fused"](render, target), 10, KERNELS)
                tk = sum(k.values())
                print(f"{key}: kernels " + ", ".join(f"{n_} {v:.3f} ms" for n_, v in sorted(k.items())) +
                      f" | {nbytes / (tk * 1e-3) / 1e9:.0f} GB/s against the algorithmic bytes", flush=True)
                rec["kernel_ms"] = k
                rec["kernel_GBps"] = nbytes / (tk * 1e-3) / 1e9
            result["loss"][key] = rec
        del render, target
        torch.cuda.empty_cache()

    if not args.no_step:
        from semantic_gaussians_b200.gaussian_model import GaussianModel
        from semantic_gaussians_b200.renderer import render_chn
        from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras

        C, W, H = 256, 1920, 1080
        scene = make_scene(1_000_000, seed=0, channels=C)
        pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
        pc.active_sh_degree = 0
        feats = torch.as_tensor(scene.features, device=dev).contiguous().requires_grad_(True)
        params = [feats, pc._xyz, pc._scaling, pc._rotation, pc._opacity]
        for p in params[1:]:
            p.requires_grad_(True)
        views = device_views(orbit_cameras(8, W, H), dev)
        bg = torch.zeros(C, device=dev)
        with torch.no_grad():                   # targets: the same scene rendered with other features, stored fp16
            other = torch.randn(feats.shape, generator=g, device=dev)
            fmaps = [render_chn(v, pc, Pipe, bg, num_channels=C, override_color=other)["render"].half() for v in views[:2]]
        it = [0]

        def step(name):
            for p in params:
                p.grad = None
            i = it[0]
            it[0] += 1
            out = render_chn(views[i % len(views)], pc, Pipe, bg, num_channels=C, override_color=feats)
            if name == "fused":
                _, grad = feature_map_loss_and_grad(out["render"], fmaps[i % 2])
                out["render"].backward(grad)
            else:
                torch_loss(out["render"], fmaps[i % 2], "cosine").backward()

        times = {"torch": [], "fused": []}
        for _ in range(args.rounds):
            for name in ("torch", "fused"):
                times[name].append(time_ms(lambda: step(name), args.step_reps, 3))
        print(f"K3-shaped step (1M Gaussians, 256 ch, 1080p, render_chn + cosine loss + backward): torch loss "
              f"{', '.join(f'{t:.2f}' for t in times['torch'])} ms | fused loss "
              f"{', '.join(f'{t:.2f}' for t in times['fused'])} ms", flush=True)
        result["step"]["k3_cosine"] = times
    print(json.dumps(result))


if __name__ == "__main__":
    main()
