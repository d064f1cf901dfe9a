"""Fusing 2D feature maps onto Gaussians: lifting by blend weights against the centre projection and the autograd route.

On the K5 shape (2 M Gaussians of the `room` scene, 512-channel fp16 maps at 640 x 480) three paths fuse the same
--views views:
  lift      fusion.lift_scene(every=1) with the fp16 maps (sgb_lift_batch: geometry, binning, alpha pass, the
            dL/dfeature contraction with the map as dL/dout, the weight-row sums; then the normalisation)
  centre    fusion.fuse_scene(depth="render", every=1): render the median depth, project every Gaussian's centre
  autograd  per view render_chn(override_color=features) forward, then .backward(map) with an fp32 copy of the map made
            before the timed region: what a user runs today to get the lift's numerator
The paths alternate --rounds times; each time ends in a device synchronise and is taken with CUDA events.  A separate
torch.profiler pass over the lift gives the time of each kernel.  Map and weight-pool bytes are computed from shapes and
the pool's chunk count.  A quality figure on synthetic data: per-Gaussian unit features f (--quality-channels) are
rendered to maps, fused by the lift and by the centre projection, and the mean cosine between the recovered features
and f is printed over the Gaussians both paths see.  Prints the card name, power limit and max SM clock, then one JSON
line."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import Pipe, device_views, gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.fusion import fuse_scene, lift_scene  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.renderer import render_chn  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, room_cameras  # noqa: E402

WCHUNK_BYTES = 16 + 16 * 8 + 16 * 256 * 4   # one 16-entry weight-pool chunk (csrc/weight_pool.cuh)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=2_000_000)
    ap.add_argument("--C", type=int, default=512)
    ap.add_argument("--W", type=int, default=640)
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--views", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--quality-channels", type=int, default=16)
    args = ap.parse_args()
    dev, gpu_name = gpu("time_lift.py")
    P, Cn, W, H, V = args.P, args.C, args.W, args.H, args.views
    scene = make_scene(P, 0, kind="room", sh=True)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs,
                                      device=dev)
    cams = room_cameras(V, W, H)
    views = device_views(cams, dev)
    for v, c in zip(views, cams):
        v.intrinsics = c.intrinsics()
    g = torch.Generator(device=dev).manual_seed(7)
    NM = 4   # device-resident maps cycled over the views (4 x 315 MB at 512 ch: more than L2 holds)
    maps16 = [torch.randn((Cn, H, W), device=dev, generator=g).half() for _ in range(NM)]
    maps32 = [m.float() for m in maps16]
    fm16 = lambda i: maps16[i % NM]   # noqa: E731
    bg3 = torch.zeros(3, device=dev)
    feats = torch.zeros((P, Cn), device=dev, requires_grad=True)
    bgC = torch.zeros(Cn, device=dev)

    def lift():
        pc.create_semantic(Cn)
        return lift_scene(pc, views, fm16, Pipe, every=1)

    def centre():
        pc.create_semantic(Cn)
        return fuse_scene(pc, views, fm16, Pipe, bg3, [W, H], depth="render", every=1)

    def autograd():
        feats.grad = None
        for i, v in enumerate(views):
            out = render_chn(v, pc, Pipe, bgC, num_channels=Cn, override_color=feats, override_shape=(W, H))
            out["render"].backward(maps32[i % NM])

    arms = {"lift": lift, "centre": centre, "autograd": autograd}
    for fn in arms.values():   # warm-up: module loads, scratch growth, pool hint
        fn()
    ctx = _lib.ctx_for(0, torch.cuda.current_stream(dev).cuda_stream)
    lift()
    torch.cuda.synchronize()
    chunks = _lib.view_stat(ctx, 1)
    t = {k: [] for k in arms}
    t0 = time.perf_counter()
    for _ in range(args.rounds):
        for k, fn in arms.items():
            t[k].append(time_ms(fn))
    for k, v in t.items():
        print(f"  {k:9s} {', '.join(f'{x:.1f}' for x in v)} ms for {V} views "
              f"({min(v) / V:.2f} ms/view best)", flush=True)
    print(f"  ({time.perf_counter() - t0:.0f} s timed)", flush=True)
    _lib.profile_enable(ctx, True)
    lift()
    stages = {k: v for k, v in _lib.profile_read(ctx).items() if v[1]}
    _lib.profile_enable(ctx, False)
    print(f"  lift stages (ms, intervals) over {V} views: {json.dumps(stages)}", flush=True)
    kt = {k: round(v, 3) for k, v in kernel_ms(lift).items()}
    print(f"  lift kernels (ms over {V} views): {json.dumps(kt)}", flush=True)
    bytes_ = {"map_fp16_per_view": Cn * H * W * 2, "map_fp32_per_view": Cn * H * W * 4,
              "pool_chunks_last_view": chunks, "pool_bytes_last_view": chunks * WCHUNK_BYTES,
              "feat_sum_bytes": P * Cn * 4}
    print(f"  bytes: {json.dumps(bytes_)}", flush=True)
    del feats, maps32

    # quality on synthetic data: render known unit features, fuse them back
    Cq = args.quality_channels
    f = torch.randn((P, Cq), device=dev, generator=g)
    f = f / f.norm(dim=1, keepdim=True)
    with torch.no_grad():
        qmaps = [render_chn(v, pc, Pipe, torch.zeros(Cq, device=dev), num_channels=Cq, override_color=f,
                            override_shape=(W, H))["render"].contiguous() for v in views]
    pc.create_semantic(Cq)
    lo = lift_scene(pc, views, qmaps, Pipe, every=1)
    lf, lm = lo["features"].clone(), lo["mask"].clone()
    pc.create_semantic(Cq)
    co = fuse_scene(pc, views, qmaps, Pipe, bg3, [W, H], depth="render", every=1)
    cf, cm = co["features"].clone(), co["mask"].clone()
    both = lm & cm
    cos = lambda x: float(torch.nn.functional.cosine_similarity(x[both], f[both], dim=1).mean()) if both.any() else None
    quality = {"seen_by_lift": int(lm.sum()), "seen_by_centre": int(cm.sum()), "seen_by_both": int(both.sum()),
               "mean_cosine_lift": cos(lf), "mean_cosine_centre": cos(cf),
               "mean_cosine_lift_all_it_sees": float(torch.nn.functional.cosine_similarity(lf[lm], f[lm], dim=1).mean())}
    print(f"  quality ({Cq} ch synthetic): {json.dumps(quality)}", flush=True)
    print(json.dumps({"card": gpu_name, "P": P, "C": Cn, "W": W, "H": H, "views": V, "ms": t, "lift_stages": stages,
                      "lift_kernels_ms": kt, "bytes": bytes_, "quality": quality}))


if __name__ == "__main__":
    main()
