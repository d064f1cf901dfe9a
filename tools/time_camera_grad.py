"""Cost of camera gradients in a training step: the K2-size step (1 M `room` Gaussians, 1920 x 1080, render() +
photometric_loss + backward) with frozen cameras against the same step with the camera tensors requiring grad, the
two arms alternating --rounds times; then a pose-only step (Gaussians frozen, CameraPoseCorrection's parameter the
only leaf); then, in a profiler pass of its own, the device time of geom_backward_kernel in each arm and of the
camera-gradient reduction's final pass.  Prints the card name, power limit and max SM clock, then one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.camera_opt import CameraPoseCorrection  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.loss_utils import photometric_loss  # noqa: E402
from semantic_gaussians_b200.renderer import render  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, room_cameras  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev, name = gpu("time_camera_grad.py")
    scene = make_scene(args.P, seed=0, kind="room", sh=True)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, scene.shs, device=dev)
    leaves = [pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest]
    bg = torch.zeros(3, device=dev)
    cams = room_cameras(8, args.width, args.height)
    views = device_views(cams, dev)
    for v, c in zip(views, cams):   # as the reference's Camera carries it (else the wrapper builds one per call)
        v.projection_matrix = torch.as_tensor(c.projection_matrix, device=dev)
    with torch.no_grad():
        gts = [render(v, pc, Pipe(), bg)["render"].clamp(0, 1).flip(-1).contiguous() for v in views]
    pose = CameraPoseCorrection(len(views), dev)
    k = [0]

    def step(cam_grad, gaussians=True):
        i = k[0] % len(views)
        k[0] += 1
        for t in leaves:
            t.requires_grad_(gaussians)
            t.grad = None
        v = pose(views[i], i) if cam_grad else views[i]
        loss, _ = photometric_loss(render(v, pc, Pipe(), bg)["render"], gts[i])
        loss.backward()
        pose.delta.grad = None

    arms = {"frozen_cameras": lambda: step(False), "camera_grads": lambda: step(True),
            "pose_only": lambda: step(True, gaussians=False)}
    res = {a: [] for a in arms}
    for a, fn in arms.items():
        time_ms(fn, reps=1, warmup=3)
    for _ in range(args.rounds):
        for a, fn in arms.items():
            res[a].append(round(time_ms(fn, reps=args.reps), 3))
    names = ["geom_backward_kernel", "camera_grad_finalize_kernel"]
    prof = {a: {n: round(ms, 4) for n, ms in kernel_ms(fn, n=8, names=names, warmup=2).items()}
            for a, fn in arms.items() if a != "pose_only"}
    print(json.dumps(dict(card=name, P=args.P, W=args.width, H=args.height, step_ms=res, kernel_ms=prof)), flush=True)


if __name__ == "__main__":
    main()
