"""Time of the optimizer step over the parameter tables of a scene: the six geometry groups of training_setup
((P,3) xyz, (P,1,3) f_dc, (P,15,3) f_rest, (P,1) opacity, (P,3) scaling, (P,4) rotation) plus a (P, C) feature table,
at 1 M x 256 (K3) and 3 M x 512 (K4).  Arms, alternated --rounds times per size and timed with CUDA events:

  torch      torch.optim.Adam, default (the foreach implementation on CUDA)
  fused      torch.optim.Adam(fused=True)
  dense      optim.GaussianAdam, every row stepped (csrc/adam.cu, one launch for the seven tables)
  view1      optim.GaussianAdam.step(visibility=...) with the visibility_filter of one view of the `room` scene
  view8      the same with the union over an 8-view batch (optim.visible_rows)

For the GaussianAdam arms a separate torch.profiler pass gives the sgb_adam_* kernel time, stated against the bytes
the step must move, computed from shapes (not measured): 28 B per element of a stepped row (p, g, m, v read; p, m, v
written) plus one mask byte per row and table, and against the H100 SXM data-sheet 3.35 TB/s.

Then a K3-shaped training step (1 M Gaussians of the blob scene, 256 channels, 1080p: render_chn + cosine
feature_map_loss_and_grad + backward + optimizer step over features, xyz, scaling, rotation, opacity) with the
torch, fused, dense and per-view-visibility arms, alternated the same way.  Each arm's optimizer lives only while it
is timed: at 3 M x 512 one set of moments is 13 GB."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.optim import GaussianAdam, visible_rows  # noqa: E402

PEAK_TBPS = 3.35
GEOMETRY = (("xyz", (3,)), ("f_dc", (1, 3)), ("f_rest", (15, 3)), ("opacity", (1,)), ("scaling", (3,)), ("rotation", (4,)))


def room_visibility(P, W, H, dev):
    """(mask of view 0, union over 8 views) of P Gaussians of the room scene."""
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.renderer import render_chn_batch
    from semantic_gaussians_b200.scene_synth import make_scene, room_cameras
    scene = make_scene(P, seed=0, kind="room")
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
    pc.active_sh_degree = 0
    with torch.no_grad():
        outs = render_chn_batch(device_views(room_cameras(8, W, H), dev), pc, Pipe, torch.zeros(8, device=dev),
                                num_channels=8, override_color=torch.rand((P, 8), device=dev))
        one, eight = visible_rows(outs[0]).clone(), visible_rows(outs).clone()
    del outs, pc
    torch.cuda.empty_cache()
    return one, eight


def make_optimizer(arm, params):
    groups = [{"params": [p], "lr": 1e-3} for p in params]
    if arm == "torch":
        return torch.optim.Adam(groups, eps=1e-15)
    if arm == "fused":
        return torch.optim.Adam(groups, eps=1e-15, fused=True)
    return GaussianAdam([dict(g, row_sparse=True) for g in groups], eps=1e-15)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--step-reps", type=int, default=10)
    ap.add_argument("--sizes", default="1000000x256x1920x1080,3000000x512x1296x968", help="PxCxWxH, comma separated")
    ap.add_argument("--no-step", action="store_true", help="skip the K3-shaped training step")
    args = ap.parse_args()
    dev, gpu_name = gpu("time_adam.py")
    result = {"card": gpu_name, "tables": {}, "step": {}}
    gen = torch.Generator(device=dev).manual_seed(0)

    for size in args.sizes.split(","):
        P, C, W, H = (int(x) for x in size.split("x"))
        one, eight = room_visibility(P, W, H, dev)
        masks = {"torch": None, "fused": None, "dense": None, "view1": one, "view8": eight}
        shapes = [(P, *s) for _, s in GEOMETRY] + [(P, C)]
        params = [torch.nn.Parameter(torch.randn(s, generator=gen, device=dev)) for s in shapes]
        for p in params:
            p.grad = torch.randn(p.shape, generator=gen, device=dev)
        row_elems = sum(p.numel() // P for p in params)
        times = {a: [] for a in masks}
        kern = {}
        for rnd in range(args.rounds):
            for arm, mask in masks.items():
                opt = make_optimizer(arm, params)
                fn = (lambda: opt.step()) if arm in ("torch", "fused") else (lambda: opt.step(visibility=mask))
                times[arm].append(time_ms(fn, args.reps, args.warmup))
                if rnd == 0 and arm not in ("torch", "fused"):
                    kern[arm] = kernel_ms(fn, 5, ["sgb_adam_"], warmup=1)["sgb_adam_"]
                del opt, fn
                torch.cuda.empty_cache()
        rec = {}
        for arm, mask in masks.items():
            frac = 1.0 if mask is None else float(mask.float().mean())
            nbytes = 28 * frac * P * row_elems + (0 if mask is None else P * len(params))
            line = f"{P} x {C} [{arm}]: " + ", ".join(f"{t:.3f}" for t in times[arm]) + " ms/step"
            rec[arm] = {"ms": times[arm], "visible_fraction": frac, "algorithmic_GB": nbytes / 1e9}
            if arm in kern:
                tbps = nbytes / (kern[arm] * 1e-3) / 1e12
                line += (f" | visible rows {100 * frac:.1f} % | sgb_adam_* kernel {kern[arm]:.3f} ms, {nbytes / 1e9:.3f} GB "
                         f"from shapes = {tbps:.2f} TB/s, {100 * tbps / PEAK_TBPS:.0f} % of {PEAK_TBPS} TB/s")
                rec[arm].update(kernel_ms=kern[arm], kernel_TBps=tbps)
            else:
                line += f" | {nbytes / 1e9:.3f} GB at 28 B/element"
            print(line, flush=True)
        result["tables"][f"{P}x{C}"] = rec
        del params, one, eight, masks
        torch.cuda.empty_cache()

    if not args.no_step:
        from semantic_gaussians_b200.gaussian_model import GaussianModel
        from semantic_gaussians_b200.renderer import render_chn
        from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
        from semantic_gaussians_b200.semantic import feature_map_loss_and_grad
        P, C, W, H = 1_000_000, 256, 1920, 1080
        scene = make_scene(P, seed=0)
        pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
        pc.active_sh_degree = 0
        feats = torch.nn.functional.normalize(torch.randn((P, C), generator=gen, device=dev), dim=1).requires_grad_(True)
        params = [feats, pc._xyz, pc._scaling, pc._rotation, pc._opacity]
        for p in params[1:]:
            p.requires_grad_(True)
        views = device_views(orbit_cameras(8, W, H), dev)
        bg = torch.zeros(C, device=dev)
        with torch.no_grad():
            other = torch.randn(feats.shape, generator=gen, device=dev)
            fmaps = [render_chn(v, pc, Pipe, bg, num_channels=C, override_color=other)["render"].half() for v in views[:2]]
            del other
        it = [0]
        fracs = []

        def step(opt, arm):
            for p in params:
                p.grad = None
            i = it[0]
            it[0] += 1
            out = render_chn(views[i % len(views)], pc, Pipe, bg, num_channels=C, override_color=feats)
            _, grad = feature_map_loss_and_grad(out["render"], fmaps[i % 2])
            out["render"].backward(grad)
            if arm == "view":
                opt.step(visibility=out["visibility_filter"])
            else:
                opt.step()

        arms = ("torch", "fused", "dense", "view")
        times = {a: [] for a in arms}
        start = [p.detach().clone() for p in params]
        for _ in range(args.rounds):
            for arm in arms:
                with torch.no_grad():                       # every arm starts from the same scene
                    for p, s in zip(params, start):
                        p.copy_(s)
                opt = make_optimizer("dense" if arm == "view" else arm, params)
                times[arm].append(time_ms(lambda: step(opt, arm), args.step_reps, 3))
                del opt
                torch.cuda.empty_cache()
        with torch.no_grad():
            for v in views:
                out = render_chn(v, pc, Pipe, bg, num_channels=C, override_color=feats)
                fracs.append(float(out["visibility_filter"].float().mean()))
        print("K3-shaped step (1M Gaussians, 256 ch, 1080p, render_chn + cosine loss + backward + optimizer step; "
              f"visible rows per view {100 * min(fracs):.1f}-{100 * max(fracs):.1f} %): " +
              " | ".join(f"{a} {', '.join(f'{t:.2f}' for t in times[a])} ms" for a in arms), flush=True)
        result["step"]["k3_cosine"] = dict(times, visible_fraction=fracs)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
