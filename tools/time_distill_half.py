"""The 3D distillation loss on a half-precision network output: semantic.voxel_feature_loss (the split forward and
gradient passes, reading and writing the output's own dtype) against the `.float()` route (an fp32 copy of the output
into voxel_feature_loss_and_grad, its fp32 gradient fed back through the cast).

  (i)  the loss alone, forward + backward, fp16 and bf16 output, on --rows rows, 60 % masked, fp16 targets:
       1536 columns with head 1 of 768 and 768 columns with head 0.  Time and the peak allocated on top of the inputs.
  (ii) one MinkUNet34A (56 -> 768) distill step (forward, loss, backward, AdamW step) on the `room` sample at --points
       Gaussians: under bf16 autocast, and under fp16 autocast with a GradScaler (the `.float()` route scales its
       gradient by scaler.get_scale(), which reads the scale on the host).

Arms alternate --rounds times; times come from CUDA events around work that ends in a synchronise.  Prints the card
name, power limit and max SM clock, then one JSON line."""
import argparse
import json
import os
import random
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from time_distill import write_room  # noqa: E402
from timing import card, time_ms  # noqa: E402

from semantic_gaussians_b200 import sparse as sp  # noqa: E402
from semantic_gaussians_b200.feature_dataset import collate_fn  # noqa: E402
from semantic_gaussians_b200.mink_unet import mink_unet  # noqa: E402
from semantic_gaussians_b200.semantic import voxel_feature_loss, voxel_feature_loss_and_grad  # noqa: E402

DEV = "cuda"
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def alternate(arms, rounds):
    """{arm: {ms_min, ms_max, peak_gib}}: each arm once to warm up, then `rounds` alternations."""
    for fn in arms.values():
        fn()
    ms = {k: [] for k in arms}
    peak = {}
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            ms[k].append(time_ms(fn))
            peak[k] = (torch.cuda.max_memory_allocated() - base) / 2**30
    return {k: {"ms_min": round(min(v), 3), "ms_max": round(max(v), 3), "peak_gib": round(peak[k], 3)}
            for k, v in ms.items()}


def loss_arms(rows, rounds, loss_type):
    res = {}
    for name, dtype in DTYPES.items():
        for F, head in ((1536, 1), (768, 0)):
            g = torch.Generator(device=DEV).manual_seed(0)
            x = torch.randn(rows, F, device=DEV, generator=g).to(dtype)
            mask = torch.rand(rows, device=DEV, generator=g) < 0.6
            gt = torch.randn(int(mask.sum()), 768, device=DEV, generator=g).half()

            # a fresh leaf per call: its half gradient is allocated inside the timed window and counted in the peak
            def split():
                xl = x.detach().requires_grad_(True)
                loss, count = voxel_feature_loss(xl, mask, gt, loss_type, head=head)
                loss.backward()

            def upcast():
                xl = x.detach().requires_grad_(True)
                loss, count, grad = voxel_feature_loss_and_grad(xl.float(), mask, gt, loss_type, head=head)
                xl.backward(grad)

            key = f"{name} {rows}x{F} head {head}"
            res[key] = alternate({"split": split, "float": upcast}, rounds)
            print("loss", key, json.dumps(res[key]), flush=True)
            del x
    return res


def step_arms(sample, rounds, loss_type):
    locs, features, features_gt, mask, head_id = collate_fn([sample])
    res = {}
    for name, dtype in DTYPES.items():
        torch.manual_seed(0)
        model = mink_unet(56, 768, arch="MinkUNet34A").to(DEV)
        opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
        scaler = torch.amp.GradScaler("cuda") if dtype == torch.float16 else None

        def forward():
            with torch.autocast("cuda", dtype=dtype):
                return model(sp.SparseTensor(features, locs))

        def step():
            if scaler is None:
                opt.step()
            else:
                scaler.step(opt)
                scaler.update()

        def split():
            out = forward()
            loss, count = voxel_feature_loss(out.F, mask, features_gt, loss_type, head_id)
            opt.zero_grad()
            (loss if scaler is None else scaler.scale(loss)).backward()
            step()

        def upcast():
            out = forward()
            loss, count, grad = voxel_feature_loss_and_grad(out.F.float(), mask, features_gt, loss_type, head_id)
            opt.zero_grad()
            out.F.backward(grad if scaler is None else grad * scaler.get_scale())
            step()

        key = f"{name}{' + GradScaler' if scaler else ''}"
        res[key] = alternate({"split": split, "float": upcast}, rounds)
        print("step", key, json.dumps(res[key]), flush=True)
        del model, opt
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loss", default="cosine", choices=["cosine", "l1", "l2"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_distill_half.py measures the GPU path and needs a GPU")
    print("card:", card(), flush=True)
    result = {"card": card(), "loss_type": args.loss}
    result["loss"] = loss_arms(args.rows, args.rounds, args.loss)
    with tempfile.TemporaryDirectory() as root:
        ds = write_room(root, args.points)
        random.seed(0)
        np.random.seed(0)
        sample = ds[0]
        result["voxels"] = int(sample[0].shape[0])
        result["step"] = step_arms(sample, args.rounds, args.loss)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
