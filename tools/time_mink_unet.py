"""MinkUNet34A (56 -> 768, the arch of the reference's distill config) on the sparse convolution of sparse.py.

Two point sets, both at voxel size 0.02:
  room      the `room` scene at --points Gaussians through voxelize_gaussians (volumetric: few neighbours per voxel)
  surface   a seeded cloud of --points points on the room's floor and four walls (1 cm jitter), closer to the
            occupancy of a scanned scene

Per set: map building (the input map, four strided maps and ten kernel maps, each with its one host read), forward,
and forward + backward in train mode, timed with CUDA events around work that ends in a synchronise, on cached maps.
The baseline replaces the native products by torch over the same pair lists (gather, mm, index_add_ per offset);
native and baseline alternate --rounds times.  A separate torch.profiler pass gives the forward kernel time of each
layer; mean pairs per output row and the FP32 rate (2 * pairs * C_in * C_out per product) come from the pair
counts.  Prints the card name, power limit and max SM clock, then one JSON line.

--dtype fp32,bf16,fp16 times each listed dtype, alternating them within every round: fp32 runs as before, bf16 / fp16
run the same fp32 model under torch.autocast("cuda", dtype) (the half-precision products).  Each dtype reports
forward, forward + backward, the peak memory allocated during forward + backward, and its own per-layer profile.  The
torch baseline runs for fp32 only (--no-baseline skips it)."""
import argparse
import contextlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import card, time_ms  # noqa: E402

from semantic_gaussians_b200 import sparse as sp  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.mink_unet import mink_unet  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, surface_voxels  # noqa: E402
from semantic_gaussians_b200.voxelize import voxelize_gaussians  # noqa: E402


def room_input(P, dev):
    scene = make_scene(P, 0, kind="room", sh=True)
    m = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs, device=dev)
    locs, feats, _ = voxelize_gaussians(m, 0.02, "all")
    return locs, feats


def torch_conv(x, kernel, km, transposed, n_out):
    """The baseline: per offset, gather the source rows, multiply, index_add_ into the destination rows."""
    out = torch.zeros((n_out, kernel.shape[2]), dtype=x.dtype, device=x.device)
    p = km.pairs.long()
    for d in range(km.K):
        a, b = km.offsets_host[d], km.offsets_host[d + 1]
        if a == b:
            continue
        src, dst = (p[a:b, 1], p[a:b, 0]) if transposed else (p[a:b, 0], p[a:b, 1])
        out = out.index_add(0, dst, x[src] @ kernel[d])
    return out


AMP = {"fp32": None, "bf16": torch.bfloat16, "fp16": torch.float16}


def amp(dt):
    """The autocast context of one timed dtype (none for fp32)."""
    return torch.autocast("cuda", dtype=AMP[dt]) if AMP[dt] else contextlib.nullcontext()


def layer_stats(model, x):
    """(name, tensor stride in, k, transposed, C_in, C_out, pairs, output rows) of every convolution, from one forward
    with hooks."""
    rows = []
    names = {m: n for n, m in model.named_modules()}

    def hook(mod, inp, out):
        xin = inp[0]
        t = xin._stride
        if mod.kernel_size == 1:
            pairs, n_out = xin.F.shape[0], xin.F.shape[0]
        elif isinstance(mod, sp.ConvolutionTranspose):
            km = xin.coordinate_manager.kernel_map(t // 2, t, 2)
            pairs, n_out = km.offsets_host[km.K], out.F.shape[0]
        else:
            km = xin.coordinate_manager.kernel_map(t, t * mod.stride, mod.kernel_size)
            pairs, n_out = km.offsets_host[km.K], out.F.shape[0]
        rows.append(dict(layer=names[mod], stride=t, k=mod.kernel_size, transposed=mod.is_transpose,
                         cin=mod.in_channels, cout=mod.out_channels, pairs=int(pairs), rows_out=int(n_out),
                         pairs_per_row=round(pairs / max(n_out, 1), 3)))

    hs = [m.register_forward_hook(hook) for m in model.modules() if isinstance(m, (sp.Convolution,
                                                                                  sp.ConvolutionTranspose))]
    with torch.no_grad():
        model(x)
    for h in hs:
        h.remove()
    return rows


def profile_layers(model, x, outdir, tag):
    """Forward kernel time of each convolution (sum of the CUDA kernels inside its record_function range)."""
    from torch.profiler import ProfilerActivity, profile, record_function
    names = {m: n for n, m in model.named_modules()}
    convs = [m for m in model.modules() if isinstance(m, (sp.Convolution, sp.ConvolutionTranspose))]
    orig = {m: m.forward for m in convs}
    for m in convs:
        def fwd(inp, _m=m):
            with record_function(f"layer:{names[_m]}"):
                return orig[_m](inp)
        m.forward = fwd
    with torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            model(x)
            torch.cuda.synchronize()
    for m in convs:
        m.forward = orig[m]
    prof.export_chrome_trace(os.path.join(outdir, f"mink_unet_{tag}.trace.json"))
    per_layer, per_kernel = {}, {}
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        if dt is None:
            dt = getattr(ev, "cuda_time_total", 0)
        if ev.key.startswith("layer:"):
            per_layer[ev.key[6:]] = dt / 1000.0
        elif ev.device_type == torch.autograd.DeviceType.CUDA or "kernel" in ev.key.lower():
            per_kernel[ev.key] = round(dt / 1000.0, 4)
    return per_layer, per_kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sets", default="room,surface")
    ap.add_argument("--dtype", default="fp32", help="comma-separated fp32, bf16, fp16: alternated in every round")
    ap.add_argument("--no-baseline", action="store_true", help="skip the torch baseline arm")
    ap.add_argument("--out", default=None, help="directory for the profiler traces and the JSON (default: a new "
                                                "temporary directory)")
    args = ap.parse_args()
    dtypes = args.dtype.split(",")
    if not dtypes or set(dtypes) - set(AMP):
        raise SystemExit(f"--dtype: comma-separated values of {sorted(AMP)}")
    if not torch.cuda.is_available():
        raise SystemExit("time_mink_unet.py needs a CUDA device")
    dev = torch.device("cuda:0")
    args.out = args.out or tempfile.mkdtemp(prefix="time_mink_unet_")
    os.makedirs(args.out, exist_ok=True)
    print(card(), flush=True)
    torch.manual_seed(0)
    model = mink_unet(56, 768, arch="MinkUNet34A").to(dev)
    result = {"card": card(), "arch": "MinkUNet34A", "points": args.points, "dtypes": dtypes, "sets": {}}
    for name in args.sets.split(","):
        locs, feats = room_input(args.points, dev) if name == "room" else surface_voxels(args.points, dev)
        M = int(locs.shape[0])

        def build_maps():
            mgr = sp.CoordinateManager(locs)
            for t in (1, 2, 4, 8, 16):
                mgr.map(t)
            mgr.kernel_map(1, 1, 5)
            for t in (1, 2, 4, 8, 16):
                mgr.kernel_map(t, t, 3)
            for t in (1, 2, 4, 8):
                mgr.kernel_map(t, 2 * t, 2)
            return mgr

        mgr = build_maps()
        t_maps = time_ms(build_maps, args.reps)
        x = sp.SparseTensor(feats, tensor_stride=1, coordinate_manager=mgr)
        model.train()

        def fwd():
            with torch.no_grad():
                model(x)

        def fwd_bwd():
            model.zero_grad(set_to_none=True)
            model(x).F.sum().backward()

        native = sp._SparseConvFunction.apply
        arms = {f"native_{dt}": {} for dt in dtypes}
        if "fp32" in dtypes and not args.no_baseline:
            arms["torch_fp32"] = {}
        for dt in dtypes:
            with amp(dt):
                fwd(), fwd_bwd()
        for _ in range(args.rounds):
            for arm in arms:
                dt = arm.split("_")[1]
                sp._SparseConvFunction.apply = native if arm.startswith("native") else torch_conv
                try:
                    with amp(dt):
                        fwd(), fwd_bwd()
                        arms[arm].setdefault("forward_ms", []).append(round(time_ms(fwd, args.reps), 3))
                        torch.cuda.reset_peak_memory_stats(dev)
                        arms[arm].setdefault("forward_backward_ms", []).append(round(time_ms(fwd_bwd, args.reps), 3))
                        arms[arm]["peak_allocated_gib"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 3)
                except torch.OutOfMemoryError:       # the baseline's autograd keeps every per-offset gather
                    arms[arm]["error"] = f"out of memory at {M} voxels"
                    model.zero_grad(set_to_none=True)
                    torch.cuda.empty_cache()
                finally:
                    sp._SparseConvFunction.apply = native
        t_e2e = time_ms(lambda: model(sp.SparseTensor(feats, locs)), args.reps)   # maps + forward, train mode, fp32
        layers = layer_stats(model, x)
        flops = sum(2 * r["pairs"] * r["cin"] * r["cout"] for r in layers)
        profiles = {}
        for dt in dtypes:
            with amp(dt):
                per_layer, per_kernel = profile_layers(model, x, args.out, f"{name}_{dt}")
            rows = []
            for r in layers:
                f = 2 * r["pairs"] * r["cin"] * r["cout"]
                ms = per_layer.get(r["layer"])
                rows.append(dict(r, fwd_kernel_ms=None if ms is None else round(ms, 4),
                                 fwd_tflops=None if not ms else round(f / ms / 1e9, 2)))
            best = min(arms[f"native_{dt}"]["forward_ms"])
            profiles[dt] = dict(forward_tflops_best=round(flops / best / 1e9, 2), layers=rows,
                                kernels_by_name=dict(sorted(per_kernel.items(), key=lambda kv: -kv[1])[:20]))
        result["sets"][name] = dict(
            voxels=M, map_build_ms=round(t_maps, 3), maps_plus_forward_ms=round(t_e2e, 3), arms=arms,
            forward_flop=flops, profiles=profiles)
        print(json.dumps({name: {k: v for k, v in result["sets"][name].items() if k != "profiles"}}), flush=True)
        for dt in dtypes:
            print(f"{name} {dt}: forward {profiles[dt]['forward_tflops_best']} TFLOP/s (best)", flush=True)
            for r in profiles[dt]["layers"]:
                print(r, flush=True)
    with open(os.path.join(args.out, "time_mink_unet.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != "sets"}), "->", args.out)


if __name__ == "__main__":
    main()
