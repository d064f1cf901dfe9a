"""Cost of depth supervision in a K2-size training step (1M Gaussians, 1920x1080, SH degree 3):

  (a) plain        render + photometric_loss + backward
  (b) in-pass      (a) with render_with_depth: expected depth E and alpha A from the same pass, plus an L1 between
                   E / max(A, eps) and a target depth on the pixels with A > 0.5
  (c) two renders  (a) plus a second C = 3 render with colours [z, 1, 0] computed in torch from means3D (the only
                   way to get a depth gradient without the option), and the same L1

timed with CUDA events (warm-up, then --reps steps over 8 orbit views), the three arms alternating --rounds times
in one run.  Prints the card name, power limit and max SM clock, then one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, time_ms  # noqa: E402

from semantic_gaussians_b200 import channel_rasterization as chn  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.loss_utils import photometric_loss  # noqa: E402
from semantic_gaussians_b200.renderer import _prepare, render, render_with_depth  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402


def depth_l1(E, A, target):
    mask = A > 0.5
    return ((E / A.clamp_min(1e-4) - target)[mask]).abs().mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev, gpu_name = gpu("time_depth.py")
    W, H = args.width, args.height

    scene = make_scene(args.P, 0, sh=True)
    m = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs, device=dev)
    params = [m._xyz, m._opacity, m._scaling, m._rotation, m._features_dc, m._features_rest]
    for p in params:
        p.requires_grad_(True)
    views = device_views(orbit_cameras(8, W, H), dev)
    bg = torch.zeros(3, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    gt = torch.rand((3, H, W), generator=g, device=dev)
    gt_depth = 2.0 + torch.rand((1, H, W), generator=g, device=dev)
    it = [0]

    def second_render(v):
        pts, common, call = _prepare(v, m, Pipe, 1.0, None, None, None, None)
        V = common["viewmatrix"].reshape(4, 4)
        z = call["means3D"] @ V[:3, 2] + V[3, 2]
        feat = torch.stack([z, torch.ones_like(z), torch.zeros_like(z)], 1)
        rs = chn.GaussianRasterizationSettings(bg=bg, debug=False, num_channels=3, **common)
        kw = {k: call[k] for k in ("means3D", "opacities", "scales", "rotations", "cov3D_precomp")}
        return chn.GaussianRasterizer(rs)(means2D=pts, colors_precomp=feat, **kw)[0]

    def step(arm):
        for p in params:
            p.grad = None
        v = views[it[0] % len(views)]
        it[0] += 1
        if arm == "in_pass":
            out = render_with_depth(v, m, Pipe, bg)
            loss = photometric_loss(out["render"], gt, 0.2, False)[0] + depth_l1(out["expected_depth"],
                                                                                   out["alpha"], gt_depth)
        else:
            out = render(v, m, Pipe, bg)
            loss = photometric_loss(out["render"], gt, 0.2, False)[0]
            if arm == "two_renders":
                ch = second_render(v)
                loss = loss + depth_l1(ch[0:1], ch[1:2], gt_depth)
        loss.backward()

    arms = ("plain", "in_pass", "two_renders")
    times = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a in arms:
            times[a].append(time_ms(lambda: step(a), args.reps, args.warmup))
    for a in arms:
        print(f"{a:12s} {', '.join(f'{t:.2f}' for t in times[a])} ms/step", flush=True)
    best = {a: min(t) for a, t in times.items()}
    print(f"depth supervision over plain (best of rounds): in-pass +{best['in_pass'] - best['plain']:.2f} ms, "
          f"two renders +{best['two_renders'] - best['plain']:.2f} ms", flush=True)
    print(json.dumps({"card": gpu_name, "P": args.P, "W": W, "H": H, "ms_per_step": times}))


if __name__ == "__main__":
    main()
