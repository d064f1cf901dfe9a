"""Time of the decoded feature-map loss and its gradients (a compact c-channel rendering lifted per pixel to the C
channels of a 2D model's feature map by a linear decoder, then the loss of distill.py:111-124):

  (a) torch   x = einsum("kc,chw->khw", W, render) + b, the reference's expressions on x against the fp16 target cast
              to fp32, gradients of render, W and b through autograd (TF32 off, torch's default)
  (b) fused   semantic_gaussians_b200.semantic.decoded_feature_map_loss_and_grads (csrc/decoder_loss.cu)

Sizes: C = 512, c = 64 at 968x1296 (K4's view) and C = 768, c = 128 at 1080x1920, fp16 targets; the two arms
alternate --rounds times per size and loss, timed with CUDA events (warm-up, then --reps repetitions).  --profile adds
a separate torch.profiler pass for the fused kernels' own time, stated against the work computed from shapes (not
measured): 6 N C c flops (decode, W^T G and G R^T; 8 N C c for cosine, which decodes twice) and N (C b_target + 8 c)
bytes (target read once, render read and its gradient written once).
Then one training step on 1M Gaussians at 968x1296 in two forms: render_chn at c = 64 + the fused decoder loss +
backward, against render_chn at C = 512 + feature_map_loss_and_grad + backward (cosine), alternating the same way."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.semantic import decoded_feature_map_loss_and_grads, feature_map_loss_and_grad  # noqa: E402

KERNELS = ("decoder_pack_kernel", "count_valid_pixels_kernel", "decoder_loss_kernel", "decoder_reduce_kernel")
LOSS_TYPES = ("cosine", "l1", "l2")


def torch_loss(x, target, loss_type):
    t = target.float()
    if loss_type == "cosine":
        m = t.norm(dim=0) > 0
        return (1 - F.cosine_similarity(x, t, dim=0))[m].mean()
    return F.l1_loss(x, t) if loss_type == "l1" else F.mse_loss(x, t)


def arms(loss_type):
    def torch_arm(render, weight, bias, target):
        x = torch.einsum("kc,chw->khw", weight, render) + bias[:, None, None]
        loss = torch_loss(x, target, loss_type)
        return (loss, *torch.autograd.grad(loss, (render, weight, bias)))

    def fused_arm(render, weight, bias, target):
        return decoded_feature_map_loss_and_grads(render, weight, target, bias=bias, loss_type=loss_type)

    return {"torch": torch_arm, "fused": fused_arm}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--step-reps", type=int, default=5)
    ap.add_argument("--no-step", action="store_true", help="skip the training step")
    ap.add_argument("--no-torch", action="store_true", help="time the fused call only")
    ap.add_argument("--profile", action="store_true", help="also report the fused kernels' time (torch.profiler)")
    args = ap.parse_args()
    dev, gpu_name = gpu("time_decoder_loss.py")
    result = {"card": gpu_name, "loss": {}, "step": {}}

    g = torch.Generator(device=dev).manual_seed(0)
    for C, c, H, W in ((512, 64, 968, 1296), (768, 128, 1080, 1920)):
        N = H * W
        render = torch.randn((c, H, W), generator=g, device=dev).requires_grad_(True)
        weight = (torch.randn((C, c), generator=g, device=dev) / c ** 0.5).requires_grad_(True)
        bias = (0.1 * torch.randn(C, generator=g, device=dev)).requires_grad_(True)
        target = torch.randn((C, H, W), generator=g, device=dev, dtype=torch.float16)
        target[:, : H // 10] = 0                                    # some empty target pixels
        nbytes = N * (C * 2 + 8 * c)
        for loss_type in LOSS_TYPES:
            fns = arms(loss_type)
            key = f"{loss_type} C={C} c={c} {H}x{W} f16"
            flops = (8 if loss_type == "cosine" else 6) * N * C * c
            names = ("fused",) if args.no_torch else ("torch", "fused")
            times = {n: [] for n in names}
            for _ in range(args.rounds):
                for name in names:
                    times[name].append(time_ms(lambda: fns[name](render, weight, bias, target), args.reps, args.warmup))
            t_f = min(times["fused"])
            line = f"{key}: fused {', '.join(f'{t:.3f}' for t in times['fused'])} ms"
            rec = {"fused_ms": times["fused"], "flops": flops, "algorithmic_GB": nbytes / 1e9}
            if not args.no_torch:
                lt = fns["torch"](render, weight, bias, target)[0]
                lf = fns["fused"](render, weight, bias, target)[0]
                line += (f" | torch {', '.join(f'{t:.3f}' for t in times['torch'])} ms | best-of speed-up "
                         f"{min(times['torch']) / t_f:.2f}x | loss torch {float(lt.detach()):.9f} fused {float(lf):.9f}")
                rec["torch_ms"] = times["torch"]
            print(line, flush=True)
            if args.profile:
                k = kernel_ms(lambda: fns["fused"](render, weight, bias, target), 5, KERNELS)
                tk = sum(k.values())
                tm = k.get("decoder_loss_kernel", float("nan"))
                print(f"{key}: kernels " + ", ".join(f"{n_} {v:.3f} ms" for n_, v in sorted(k.items())) +
                      f" | main kernel {flops / (tm * 1e-3) / 1e12:.1f} TFLOP/s FP32 and "
                      f"{nbytes / (tm * 1e-3) / 1e9:.0f} GB/s against the shapes' work", flush=True)
                rec["kernel_ms"] = k
                rec["main_TFLOPs"] = flops / (tm * 1e-3) / 1e12
                rec["main_GBps"] = nbytes / (tm * 1e-3) / 1e9
            result["loss"][key] = rec
        del render, weight, bias, target
        torch.cuda.empty_cache()

    if not args.no_step:
        from semantic_gaussians_b200.gaussian_model import GaussianModel
        from semantic_gaussians_b200.renderer import render_chn
        from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras

        C, c, W, H = 512, 64, 1296, 968
        scene = make_scene(1_000_000, seed=0, channels=c)
        pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
        pc.active_sh_degree = 0
        P = scene.xyz.shape[0]
        compact = torch.as_tensor(scene.features, device=dev).contiguous().requires_grad_(True)
        wide = torch.randn((P, C), generator=g, device=dev).requires_grad_(True)
        decoder = torch.nn.Linear(c, C, device=dev)
        geo = [pc._xyz, pc._scaling, pc._rotation, pc._opacity]
        for p in geo:
            p.requires_grad_(True)
        views = device_views(orbit_cameras(8, W, H), dev)
        with torch.no_grad():                   # targets: the same scene rendered with other 512-ch features, fp16
            other = torch.randn((P, C), generator=g, device=dev)
            fmaps = [render_chn(v, pc, Pipe, torch.zeros(C, device=dev), num_channels=C,
                                override_color=other)["render"].half() for v in views[:2]]
            del other
        bg_c, bg_w = torch.zeros(c, device=dev), torch.zeros(C, device=dev)
        it = [0]

        def step(name):
            for p in geo + [compact, wide, decoder.weight, decoder.bias]:
                p.grad = None
            i = it[0]
            it[0] += 1
            v = views[i % len(views)]
            if name == "compact":
                out = render_chn(v, pc, Pipe, bg_c, num_channels=c, override_color=compact)
                _, g_r, g_w, g_b = decoded_feature_map_loss_and_grads(out["render"], decoder.weight, fmaps[i % 2],
                                                                      bias=decoder.bias)
                out["render"].backward(g_r)
                decoder.weight.grad, decoder.bias.grad = g_w, g_b
            else:
                out = render_chn(v, pc, Pipe, bg_w, num_channels=C, override_color=wide)
                _, grad = feature_map_loss_and_grad(out["render"], fmaps[i % 2])
                out["render"].backward(grad)

        times = {"wide": [], "compact": []}
        for _ in range(args.rounds):
            for name in ("wide", "compact"):
                times[name].append(time_ms(lambda: step(name), args.step_reps, 2))
        print(f"training step (1M Gaussians, {W}x{H}, cosine): render_chn C={C} + feature_map_loss_and_grad + backward "
              f"{', '.join(f'{t:.2f}' for t in times['wide'])} ms | render_chn c={c} + decoded loss + backward "
              f"{', '.join(f'{t:.2f}' for t in times['compact'])} ms", flush=True)
        result["step"]["k4_view_cosine"] = times
    print(json.dumps(result))


if __name__ == "__main__":
    main()
