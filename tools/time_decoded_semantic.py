"""Time of the semantic head of a compact field through its linear decoder (a c-channel rendering lifted per pixel to
the C channels of the text embeddings by x = W r + b), three arms alternated --rounds times per size:

  (a) torch   x = einsum("kc,chw->khw", W, render) + b, then semantic_head(x, text): the (C,H,W) image is written
              and read back
  (b) fused   semantic_gaussians_b200.semantic.decoded_semantic_head, sim + label (csrc/decoded_head.cu)
  (c) label   decoded_semantic_head(..., return_sim=False): no norm, no K planes

Sizes: C = 512, c = 64 at 968x1296 and C = 768, c = 128 at 1080x1920, K = 21 and 201.  Each arm reports its mean ms
over --reps calls after --warmup, and the peak allocated memory above the inputs in a call of its own.  A separate
torch.profiler pass gives the fused kernels' device time, stated against the work computed from shapes (not measured):
K c FMAs per pixel for the numerators, c^2 float64 FMAs per pixel for the norm (sim only), 4 c bytes read and 4 K + 8
bytes written per pixel.  Then one evaluation view on 1 M Gaussians at 968x1296 (C = 512, c = 64, K = 21):
render_chn(c) + arm (a), render_chn(c) + arm (c), and the logit render render_semantic_labels(logits =
decoded_feature_logits(...)), alternated the same way."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.semantic import (decoded_feature_logits, decoded_semantic_head,  # noqa: E402
                                              render_semantic_labels, semantic_head)

KERNELS = ("decoded_head_prologue_kernel", "decoded_head_kernel")


def torch_arm(render, weight, bias, text):
    x = torch.einsum("kc,chw->khw", weight, render) + bias[:, None, None]
    return semantic_head(x, text)


def fused_arm(render, weight, bias, text):
    return decoded_semantic_head(render, weight, text, bias=bias)


def label_arm(render, weight, bias, text):
    return decoded_semantic_head(render, weight, text, bias=bias, return_sim=False)


ARMS = {"torch": torch_arm, "fused": fused_arm, "label": label_arm}


def peak_mib(fn):
    """Peak allocated MiB above what was allocated before one call of fn (its outputs included)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    del out
    return peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=1_000_000, help="scene size of the evaluation view")
    ap.add_argument("--no-view", action="store_true", help="skip the evaluation view")
    args = ap.parse_args()
    dev, gpu_name = gpu("time_decoded_semantic.py")
    result = {"card": gpu_name, "head": {}, "view": {}}

    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():
        for C, c, H, W in ((512, 64, 968, 1296), (768, 128, 1080, 1920)):
            N = H * W
            render = torch.randn((c, H, W), generator=g, device=dev)
            weight = torch.randn((C, c), generator=g, device=dev) / c ** 0.5
            bias = 0.1 * torch.randn(C, generator=g, device=dev)
            for K in (21, 201):
                text = torch.nn.functional.normalize(torch.randn((K, C), generator=g, device=dev), dim=1)
                key = f"C={C} c={c} K={K} {H}x{W}"
                times = {n: [] for n in ARMS}
                for _ in range(args.rounds):
                    for name, fn in ARMS.items():
                        times[name].append(time_ms(lambda: fn(render, weight, bias, text), args.reps, args.warmup))
                peaks = {name: peak_mib(lambda: fn(render, weight, bias, text)) for name, fn in ARMS.items()}
                s_t, l_t = torch_arm(render, weight, bias, text)
                s_f, l_f = fused_arm(render, weight, bias, text)
                agree = float((l_t == l_f).float().mean())
                dsim = float((s_t - s_f).abs().max())
                k_f = kernel_ms(lambda: fused_arm(render, weight, bias, text), 5, KERNELS)
                k_l = kernel_ms(lambda: label_arm(render, weight, bias, text), 5, KERNELS)
                fma32, fma64 = N * K * c, N * c * c
                t_kf, t_kl = k_f.get("decoded_head_kernel", float("nan")), k_l.get("decoded_head_kernel", float("nan"))
                rates = {
                    "sim_label_TFLOPs_fp32": 2 * fma32 / (t_kf * 1e-3) / 1e12,
                    "sim_label_TFLOPs_fp64": 2 * fma64 / (t_kf * 1e-3) / 1e12,
                    "sim_label_GBps": N * (4 * c + 4 * K + 8) / (t_kf * 1e-3) / 1e9,
                    "label_TFLOPs_fp32": 2 * fma32 / (t_kl * 1e-3) / 1e12,
                    "label_GBps": N * (4 * c + 8) / (t_kl * 1e-3) / 1e9,
                }
                print(f"{key}: " + " | ".join(f"{n} {', '.join(f'{t:.3f}' for t in ts)} ms, peak {peaks[n]:.0f} MiB"
                                             for n, ts in times.items()) +
                      f" | labels equal {agree:.6f}, max |sim diff| {dsim:.2e}", flush=True)
                print(f"{key}: kernels sim+label " + ", ".join(f"{n} {v:.3f} ms" for n, v in sorted(k_f.items())) +
                      " | label only " + ", ".join(f"{n} {v:.3f} ms" for n, v in sorted(k_l.items())) +
                      f" | main kernel against the shapes' work: sim+label {rates['sim_label_TFLOPs_fp32']:.1f} "
                      f"TFLOP/s fp32 + {rates['sim_label_TFLOPs_fp64']:.1f} TFLOP/s fp64, "
                      f"{rates['sim_label_GBps']:.0f} GB/s; label {rates['label_TFLOPs_fp32']:.1f} TFLOP/s fp32, "
                      f"{rates['label_GBps']:.0f} GB/s", flush=True)
                result["head"][key] = {"ms": times, "peak_MiB": peaks, "kernel_ms_sim_label": k_f,
                                       "kernel_ms_label": k_l, "rates_from_shapes": rates, "label_agreement": agree,
                                       "max_abs_sim_diff": dsim}
                del s_t, l_t, s_f, l_f, text
            del render, weight, bias
            torch.cuda.empty_cache()

        if not args.no_view:
            from semantic_gaussians_b200.gaussian_model import GaussianModel
            from semantic_gaussians_b200.renderer import render_chn
            from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras

            C, c, K, W, H = 512, 64, 21, 1296, 968
            scene = make_scene(args.gaussians, seed=0, channels=c)
            pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
            pc.active_sh_degree = 0
            f = torch.as_tensor(scene.features, device=dev).contiguous()
            weight = torch.randn((C, c), generator=g, device=dev) / c ** 0.5
            bias = 0.1 * torch.randn(C, generator=g, device=dev)
            text = torch.nn.functional.normalize(torch.randn((K, C), generator=g, device=dev), dim=1)
            bg_c = torch.zeros(c, device=dev)
            bg_w = weight @ bg_c + bias
            views = device_views(orbit_cameras(8, W, H), dev)
            logits = decoded_feature_logits(f, weight, text, bias, pad_to=4)
            it = [0]

            def view():
                i = it[0]
                it[0] += 1
                return views[i % len(views)]

            def render_torch():
                r = render_chn(view(), pc, Pipe, bg_c, num_channels=c, override_color=f)["render"]
                return torch_arm(r, weight, bias, text)[1]

            def render_label():
                r = render_chn(view(), pc, Pipe, bg_c, num_channels=c, override_color=f)["render"]
                return label_arm(r, weight, bias, text)[1]

            def logit_render():
                return render_semantic_labels(view(), pc, Pipe, bg_w, text, logits=logits)["label"]

            view_arms = {"render_chn + torch decode + semantic_head": render_torch,
                         "render_chn + decoded_semantic_head label only": render_label,
                         "render_semantic_labels on decoded_feature_logits": logit_render}
            times = {n: [] for n in view_arms}
            for _ in range(args.rounds):
                for name, fn in view_arms.items():
                    times[name].append(time_ms(fn, args.reps, args.warmup))
            peaks = {name: peak_mib(fn) for name, fn in view_arms.items()}
            t_logits = time_ms(lambda: decoded_feature_logits(f, weight, text, bias, pad_to=4), args.reps, args.warmup)
            it[0] = 0
            la = render_torch()
            it[0] = 0
            lb = logit_render()
            agree = float((la == lb).float().mean())
            print(f"evaluation view ({args.gaussians} Gaussians, {W}x{H}, C={C} c={c} K={K}): " +
                  " | ".join(f"{n} {', '.join(f'{t:.3f}' for t in ts)} ms, peak {peaks[n]:.0f} MiB"
                             for n, ts in times.items()) +
                  f" | decoded_feature_logits once per scene {t_logits:.3f} ms | logit-render labels equal to the "
                  f"render-then-decode labels at {agree:.6f} of the pixels", flush=True)
            result["view"] = {"ms": times, "peak_MiB": peaks, "decoded_feature_logits_ms": t_logits,
                              "label_agreement": agree}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
