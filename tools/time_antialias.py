"""Cost of anti-aliasing (pipe.antialiasing): the K2-size step (1 M `room` Gaussians, 1920 x 1080, render() +
photometric_loss + backward) and a K3-shape render_chn step (256 channels, loss sum(render * target) + backward), each
with the flag off and on, the arms alternating --rounds times; then, in a profiler pass of its own, the device time of
preprocess_kernel and geom_backward_kernel in each arm of the K2 step.  Prints the card name, power limit and max SM
clock, then one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.loss_utils import photometric_loss  # noqa: E402
from semantic_gaussians_b200.renderer import render, render_chn  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, room_cameras  # noqa: E402


class AAPipe(Pipe):
    antialiasing = True


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--channels", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev, name = gpu("time_antialias.py")
    scene = make_scene(args.P, seed=0, kind="room", sh=True)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, scene.shs, device=dev)
    leaves = [pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest]
    for t in leaves:
        t.requires_grad_(True)
    feats = torch.randn((args.P, args.channels), device=dev).requires_grad_(True)
    bg, bgc = torch.zeros(3, device=dev), torch.zeros(args.channels, device=dev)
    cams = room_cameras(8, args.width, args.height)
    views = device_views(cams, dev)
    with torch.no_grad():
        gts = [render(v, pc, Pipe(), bg)["render"].clamp(0, 1).flip(-1).contiguous() for v in views]
    target = torch.randn((args.channels, args.height, args.width), device=dev)
    k = [0]

    def step(pipe, chn):
        i = k[0] % len(views)
        k[0] += 1
        for t in leaves + [feats]:
            t.grad = None
        if chn:
            out = render_chn(views[i], pc, pipe, bgc, num_channels=args.channels, override_color=feats)["render"]
            (out * target).sum().backward()
        else:
            loss, _ = photometric_loss(render(views[i], pc, pipe, bg)["render"], gts[i])
            loss.backward()

    arms = {"k2_off": lambda: step(Pipe(), False), "k2_on": lambda: step(AAPipe(), False),
            "k3_off": lambda: step(Pipe(), True), "k3_on": lambda: step(AAPipe(), True)}
    res = {a: [] for a in arms}
    for a, fn in arms.items():
        time_ms(fn, reps=1, warmup=3)
    for _ in range(args.rounds):
        for a, fn in arms.items():
            res[a].append(round(time_ms(fn, reps=args.reps), 3))
    names = ["preprocess_kernel", "geom_backward_kernel"]
    prof = {a: {n: round(ms, 4) for n, ms in kernel_ms(arms[a], n=8, names=names, warmup=2).items()}
            for a in ("k2_off", "k2_on")}
    print(json.dumps(dict(card=name, P=args.P, W=args.width, H=args.height, C=args.channels, step_ms=res,
                          kernel_ms=prof)), flush=True)


if __name__ == "__main__":
    main()
