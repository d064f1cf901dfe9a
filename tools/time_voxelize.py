"""Voxelizing a Gaussian scene for the 3D network: the device path against the reference's host round trip.

  device   voxelize_gaussians(model, voxel_size): sgb_voxelize, the feature gather and the normal rotation on the GPU,
           one read of M back to the host
  host     what eval_segmentation.py / distill.py do: get_locs_and_features() (copies to the host), the voxelization
           in numpy (the in-repo oracle, the reference's own arithmetic), and the upload of locs, features and vox_ind

Both arms end in a device synchronise and are timed with CUDA events, alternating --rounds times at each P.  Outputs of
the two arms are compared bit for bit first.  A separate torch.profiler pass over the device arm gives the time of each
kernel.  Prints the card name, power limit and max SM clock, then one JSON line."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from timing import gpu, kernel_ms, time_ms  # noqa: E402

from oracle import voxel_oracle as vo  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene  # noqa: E402
from semantic_gaussians_b200.voxelize import voxelize_gaussians  # noqa: E402


def host_round_trip(m, voxel_size, dev):
    locs, feats = m.get_locs_and_features("all")
    first, _, coords, _ = vo.voxelize(locs, np.diag([1 / voxel_size] * 3 + [1.0]))
    feats = vo.rotate_normals(feats[first], np.eye(3))
    locs_t = torch.from_numpy(coords.astype(np.int32))
    locs_t = torch.cat([torch.ones(locs_t.shape[0], 1, dtype=torch.int), locs_t], dim=1).to(dev)
    return locs_t, torch.from_numpy(feats).float().to(dev), torch.from_numpy(first).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--voxel-size", type=float, default=0.02)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev, gpu_name = gpu("time_voxelize.py")
    result = {"card": gpu_name, "voxel_size": args.voxel_size, "sizes": {}}
    for P in args.P:
        scene = make_scene(P, 0, kind="room", sh=True)
        m = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs,
                                         device=dev)
        dev_arm = lambda: voxelize_gaussians(m, args.voxel_size)             # noqa: E731
        host_arm = lambda: host_round_trip(m, args.voxel_size, dev)          # noqa: E731
        a, b = dev_arm(), host_arm()
        same = all(torch.equal(x, y) for x, y in zip(a, b))
        M = int(a[2].shape[0])
        print(f"P={P}: M={M} voxels, device == host: {same}", flush=True)
        if not same:
            raise SystemExit("device and host arms disagree")
        t = {"device": [], "host": []}
        t0 = time.perf_counter()
        for _ in range(args.rounds):
            t["device"].append(time_ms(dev_arm, args.reps))
            t["host"].append(time_ms(host_arm, args.host_reps))
        for k, v in t.items():
            print(f"  {k:7s} {', '.join(f'{x:.3f}' for x in v)} ms/call", flush=True)
        best = {k: min(v) for k, v in t.items()}
        print(f"  host / device (best of rounds): {best['host'] / best['device']:.0f}x "
              f"({time.perf_counter() - t0:.0f} s timed)", flush=True)
        kt = {k: round(v, 4) for k, v in kernel_ms(dev_arm, args.reps, warmup=1).items()}
        print(f"  kernels (ms per call): {json.dumps(kt)}", flush=True)
        result["sizes"][P] = {"M": M, "ms_per_call": t, "kernel_ms_per_call": kt}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
