"""The 3D distillation step of distill.py with config/distill_scannet.yaml's aug: True, on the device.

  (i)   one FeatureDataset(aug=True) sample of the synthetic `room` scene (8 x 8 x 3 m) at --points Gaussians, read
        from a page-cached PLY and fused-feature file: the device path (feature_dataset.FeatureDataset[0]) against
        the host restatement (numpy elastic distortion of oracle/augment_oracle.py with the same scipy noise, the
        numpy voxelization of oracle/voxel_oracle.py, numpy gathers and flip) plus the upload of its four tensors.
  (ii)  the loss and its gradient on M = --rows rows x 1536 columns (head 1 of 768), 60 % masked, fp16 targets:
        semantic.voxel_feature_loss_and_grad against distill.py's torch expression and autograd, with the peak
        memory each arm allocates on top of its inputs.
  (iii) one MinkUNet34A (56 -> 768) distill step on the 1 M `room` sample: forward, loss, backward, AdamW step,
        with the fused loss and with the torch loss.

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
from timing import card, time_ms  # noqa: E402

from oracle import augment_oracle as ao  # noqa: E402
from oracle import voxel_oracle as vo  # noqa: E402
from semantic_gaussians_b200 import sparse as sp  # noqa: E402
from semantic_gaussians_b200.feature_dataset import FeatureDataset, collate_fn  # noqa: E402
from semantic_gaussians_b200.gaussian_model import GaussianModel  # noqa: E402
from semantic_gaussians_b200.io_formats import read_vertex_ply, save_fused_features, save_gaussian_ply  # noqa: E402
from semantic_gaussians_b200.mink_unet import mink_unet  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene  # noqa: E402
from semantic_gaussians_b200.semantic import voxel_feature_loss_and_grad  # noqa: E402
from semantic_gaussians_b200.voxelize import distill_targets  # noqa: E402

DEV = "cuda"


def write_room(root, P):
    scene = make_scene(P, 0, kind="room", sh=True)
    m = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs,
                                     device="cpu")
    save_gaussian_ply(os.path.join(root, "g", "room", "point_cloud", "iteration_30000", "point_cloud.ply"), m)
    g = torch.Generator().manual_seed(1)
    mask = torch.rand(P, generator=g) < 0.6
    save_fused_features(os.path.join(root, "p", "room", "feat_0.pt"), torch.randn(int(mask.sum()), 768, generator=g),
                        mask)
    return FeatureDataset(os.path.join(root, "g"), os.path.join(root, "p"), 30000, 0.02, True, "all")


def host_sample(ds):
    """FeatureDataset[0] restated on the host (numpy / scipy / CPU torch) and uploaded."""
    ply, pt, head_id = ds.data[0]
    el = read_vertex_ply(ply)
    xyz = np.stack((el["x"], el["y"], el["z"]), axis=1)
    idx = lambda p: sorted((k for k in el if k.startswith(p)), key=lambda k: int(k.split("_")[-1]))  # noqa: E731
    names = ["opacity", "f_dc_0", "f_dc_1", "f_dc_2"] + idx("f_rest_") + idx("scale_") + idx("rot")
    feats = np.stack([el[n] for n in names], axis=1).astype(np.float64)
    gt = torch.load(pt)
    xyz, _ = ao.elastic_distortion_all(xyz, ds.ELASTIC_DISTORT_PARAMS)
    M_v, M_r = ds.voxelizer.get_transformation_matrix()
    first, _, coords, _ = vo.voxelize(xyz, M_r @ M_v)
    f = feats[first]
    f[:, 3:6] = f[:, 3:6] @ M_r[:3, :3].T
    mask, features_gt = distill_targets(torch.from_numpy(first), gt["mask_full"], gt["feat"])
    if random.random() < 0.95:
        for axis in (0, 1):
            if random.random() < 0.5:
                coords[:, axis] = coords[:, axis].max() - coords[:, axis]
    locs = np.concatenate([np.ones((len(coords), 1), np.int64), coords], axis=1).astype(np.int32)
    return (torch.from_numpy(locs).to(DEV), torch.from_numpy(f.astype(np.float32)).to(DEV), features_gt.to(DEV),
            mask.to(DEV), head_id)


def torch_loss(output, mask, gt, loss_type, head, C=768):
    o = output[mask]
    y = gt.float()
    if loss_type == "cosine":
        nm = y.norm(dim=-1) > 0
        return (1 - torch.nn.CosineSimilarity()(o[nm][:, head * C:(head + 1) * C], y[nm])).mean()
    return (torch.nn.L1Loss() if loss_type == "l1" else torch.nn.MSELoss())(o[:, head * C:(head + 1) * C], y)


def loss_arms(rows, rounds):
    g = torch.Generator(device=DEV).manual_seed(0)
    out = torch.randn(rows, 1536, device=DEV, generator=g)
    mask = torch.rand(rows, device=DEV, generator=g) < 0.6
    gt = torch.randn(int(mask.sum()), 768, device=DEV, generator=g).half()

    def fused(lt):
        loss, count, grad = voxel_feature_loss_and_grad(out, mask, gt, lt, head=1)
        return loss

    def autograd(lt):
        x = out.detach().requires_grad_(True)
        loss = torch_loss(x, mask, gt, lt, 1)
        loss.backward()
        return loss

    res = {}
    for lt in ("cosine", "l1", "l2"):
        arms = {"fused": fused, "torch": autograd}
        for fn in arms.values():
            fn(lt)
        ms = {k: [] for k in arms}
        peak = {}
        for _ in range(rounds):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                ms[k].append(time_ms(lambda: fn(lt)))
                peak[k] = (torch.cuda.max_memory_allocated() - base) / 2**30
        res[lt] = {k: {"ms_min": min(v), "ms_max": max(v), "peak_gib": round(peak[k], 3)} for k, v in ms.items()}
        print(lt, json.dumps(res[lt]), flush=True)
    return res


def step_arms(sample, rounds):
    locs, features, features_gt, mask, head_id = collate_fn([sample])
    torch.manual_seed(0)
    model = mink_unet(56, 768, arch="MinkUNet34A").to(DEV)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
    res = {}
    for lt in ("cosine", "l1", "l2"):
        def fused():
            out = model(sp.SparseTensor(features, locs))
            loss, count, grad = voxel_feature_loss_and_grad(out.F, mask, features_gt, lt, head_id)
            opt.zero_grad()
            out.F.backward(grad)
            opt.step()

        def autograd():
            out = model(sp.SparseTensor(features, locs))
            loss = torch_loss(out.F, mask, features_gt, lt, head_id)
            opt.zero_grad()
            loss.backward()
            opt.step()

        arms = {"fused": fused, "torch": autograd}
        for fn in arms.values():
            fn()
        ms = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                ms[k].append(time_ms(fn))
        res[lt] = {k: {"ms_min": min(v), "ms_max": max(v)} for k, v in ms.items()}
        print("step", lt, json.dumps(res[lt]), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_distill.py measures the GPU path and needs a GPU")
    print("card:", card(), flush=True)
    result = {"card": card(), "sample": {}}
    with tempfile.TemporaryDirectory() as root:
        first_sample = None
        for P in args.points:
            ds = write_room(os.path.join(root, str(P)), P)
            arms = {"device": lambda: ds[0], "host": lambda: host_sample(ds)}
            for k, fn in arms.items():       # warm-up; also checks that both arms give the same sample
                random.seed(0)
                np.random.seed(0)
                got = fn()
                if k == "device":
                    want = got
                else:
                    assert all(torch.equal(a, b) for a, b in zip(want[:4], got[:4])), "host and device samples differ"
            ms = {k: [] for k in arms}
            s = [None]                       # the last sample, kept until the next one replaces it
            for r in range(args.rounds):
                for k, fn in arms.items():
                    random.seed(r)
                    np.random.seed(r)
                    ms[k].append(time_ms(lambda: s.__setitem__(0, fn())))
                    if k == "device" and first_sample is None:
                        first_sample = s[0]
            result["sample"][P] = {"voxels": int(want[0].shape[0]),
                                   **{k: {"ms_min": min(v), "ms_max": max(v)} for k, v in ms.items()}}
            print("sample", P, json.dumps(result["sample"][P]), flush=True)
            del ds
        result["loss"] = loss_arms(args.rows, args.rounds)
        result["step"] = step_arms(first_sample, args.rounds)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
