"""Cost of a joint colour + feature training step (forward and backward of one view) three ways:

  joint      render_with_features: one geometry pass and one binning for the RGB image and the (c, H, W) feature image
             (for c > 4 one walk of the tile lists: the "alpha_pass" stage is also the RGB blend)
  separate   render() + render_chn() on the same inputs: two geometry passes, two binnings, two geometry backwards
  concat     SH colours evaluated in torch (convert_shs_python), [rgb | features] rendered through one render_chn
             with c + 3 channels (no median depth; RGB within rounding of render(), not bitwise)

Every arm takes the fused photometric loss on the RGB image and a fixed random dL/d feature image, in one backward.
Timed with CUDA events (warm-up, then --reps steps over 8 room views), the arms alternating --rounds times in one run;
then, per arm, one step with the library's stage tracing (sgb_profile_*) and the peak memory of one step.  Prints the
card name, power limit and max SM clock, then one JSON line per size."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, time_ms  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.loss_utils import photometric_loss  # noqa: E402
from semantic_gaussians_b200.renderer import _prepare, render, render_chn, render_with_features  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, room_cameras  # noqa: E402


class PySHPipe(Pipe):
    convert_shs_python = True


def parse_size(s):
    wh, c = s.split(":")
    w, h = wh.split("x")
    return int(w), int(h), int(c)


def run_size(m, params, dev, W, H, c, args):
    views = device_views(room_cameras(8, W, H), dev)
    g = torch.Generator(device=dev).manual_seed(0)
    feats = torch.randn((m._xyz.shape[0], c), generator=g, device=dev).requires_grad_(True)
    bg, bgf = torch.zeros(3, device=dev), torch.zeros(c, device=dev)
    gt = torch.rand((3, H, W), generator=g, device=dev)
    g_feat = torch.randn((c, H, W), generator=g, device=dev) * 1e-3
    it = [0]

    def step(arm):
        for p in params + [feats]:
            p.grad = None
        v = views[it[0] % len(views)]
        it[0] += 1
        if arm == "joint":
            out = render_with_features(v, m, Pipe, bg, feats, bgf)
            rgb, fimg = out["render"], out["features"]
        elif arm == "separate":
            rgb = render(v, m, Pipe, bg)["render"]
            fimg = render_chn(v, m, Pipe, bgf, num_channels=c, override_color=feats)["render"]
        else:
            _, _, call = _prepare(v, m, PySHPipe, 1.0, None, None, None, None)
            both = torch.cat((call["colors_precomp"], feats), 1)
            img = render_chn(v, m, Pipe, torch.cat((bg, bgf)), num_channels=c + 3, override_color=both)["render"]
            rgb, fimg = img[:3], img[3:]
        loss = photometric_loss(rgb, gt, 0.2, False)[0]
        torch.autograd.backward([loss, fimg], [None, g_feat])

    arms = ("joint", "separate", "concat")
    for a in arms:
        step(a)
    times = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a in arms:
            times[a].append(time_ms(lambda: step(a), args.reps, args.warmup))
    ctx = _lib.ctx_for(dev.index or 0, torch.cuda.current_stream(dev).cuda_stream)
    stages, peak = {}, {}
    for a in arms:
        _lib.profile_enable(ctx, True)
        step(a)
        torch.cuda.synchronize()
        stages[a] = {k: round(ms, 3) for k, (ms, n) in _lib.profile_read(ctx).items() if n}
        _lib.profile_enable(ctx, False)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        step(a)
        torch.cuda.synchronize()
        peak[a] = round((torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20, 1)
    del feats, gt, g_feat
    for a in arms:
        print(f"{W}x{H} c={c} {a:9s} {', '.join(f'{t:.2f}' for t in times[a])} ms/step, peak +{peak[a]} MiB, "
              f"stages {stages[a]}", flush=True)
    return {"W": W, "H": H, "c": c, "ms_per_step": times, "peak_mib_over_model": peak, "stage_ms": stages}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--sizes", nargs="+", default=["1920x1080:64", "1296x968:512"],
                    help="WxH:c, one timed workload each")
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    sizes = [parse_size(s) for s in args.sizes]
    dev, gpu_name = gpu("time_joint.py")
    scene = make_scene(args.P, 0, kind="room", sh=True)
    m = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs, device=dev)
    params = [m._xyz, m._opacity, m._scaling, m._rotation, m._features_dc, m._features_rest]
    for p in params:
        p.requires_grad_(True)
    for W, H, c in sizes:
        res = run_size(m, params, dev, W, H, c, args)
        print(json.dumps(dict(card=gpu_name, P=args.P, scene="room", **res)), flush=True)


if __name__ == "__main__":
    main()
