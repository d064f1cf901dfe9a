"""Nearest-point label transfer for a per-point 3D evaluation: `nearest_points` against the two ways a user has without
it.

  nearest_points   sgb_nearest on the GPU (exact, fp32)
  cdist            chunked torch.cdist + argmin on the GPU (brute force; cdist's matrix-product form rounds
                   differently, so its index is compared, not required to be equal)
  ckdtree          scipy.spatial.cKDTree(ref).query(q, workers=-1) on the host, with the download of both sets, the
                   tree build and the upload of the index included

References: the scene_synth `room` scene (volumetric Gaussians in 8 x 8 x 3 m); queries: points sampled on the room's
floor and walls (`surface_points`), as scan vertices would be.  Every arm ends in a device synchronise and is timed
with CUDA events; nearest_points over --reps calls per round, the others once per round.  A separate torch.profiler
pass gives nearest_points' kernel times.  Prints the card name, power limit and max SM clock, the host core count,
then one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from timing import gpu, kernel_ms, time_ms  # noqa: E402

from semantic_gaussians_b200.metric import nearest_points  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, surface_points  # noqa: E402


def cdist_arm(q, r, chunk_elems=1 << 31):
    step = max(1, chunk_elems // r.shape[0])
    return torch.cat([torch.cdist(q[s:s + step], r).argmin(1) for s in range(0, q.shape[0], step)])


def ckdtree_arm(q, r):
    from scipy.spatial import cKDTree
    _, j = cKDTree(r.cpu().numpy()).query(q.cpu().numpy(), workers=-1)
    return torch.from_numpy(j).to(q.device)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[1_000_000, 3_000_000], help="reference (Gaussian) counts")
    ap.add_argument("--M", type=int, nargs="+", default=[150_000, 1_000_000], help="query (surface point) counts")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arms", nargs="+", default=["nearest_points", "cdist", "ckdtree"])
    args = ap.parse_args()
    dev, gpu_name = gpu("time_nearest.py")
    cores = os.cpu_count()
    print(f"host cores (cKDTree workers=-1): {cores}", flush=True)
    result = {"card": gpu_name, "host_cores": cores, "sizes": {}}
    for P in args.P:
        r = torch.from_numpy(make_scene(P, 0, kind="room").xyz).to(dev)
        for M in args.M:
            q = torch.from_numpy(surface_points(M, 1)).to(dev)
            arms = {"nearest_points": lambda: nearest_points(q, r)[0], "cdist": lambda: cdist_arm(q, r),
                    "ckdtree": lambda: ckdtree_arm(q, r)}
            arms = {k: arms[k] for k in args.arms}
            index = nearest_points(q, r)[0]                     # the first calls also warm every arm up
            agree = {k: float((fn() == index).float().mean()) for k, fn in arms.items() if k != "nearest_points"}
            t = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    t[k].append(round(time_ms(fn, args.reps if k == "nearest_points" else 1), 3))
            kt = {k: round(v, 4) for k, v in kernel_ms(lambda: nearest_points(q, r), args.reps, warmup=1).items()}
            print(f"P={P} M={M}: ms per call {json.dumps(t)}; index agreement with nearest_points {json.dumps(agree)}",
                  flush=True)
            print(f"  nearest_points kernels (ms per call): {json.dumps(kt)}", flush=True)
            result["sizes"][f"{P}x{M}"] = {"ms_per_call": t, "agreement": agree, "kernel_ms_per_call": kt}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
