"""Generates tests/golden/distill_golden.npz by running the REFERENCE's own augmentation and dataset code
(dataset/augmentation.py ElasticDistortion, dataset/fusion_utils.py Voxelizer, dataset/feature_dataset.py
FeatureDataset.__getitem__, imported from /root/reference as make_voxel_golden.py imports fusion_utils.py) on seeded
synthetic scenes.  Run in the build container:

    python tests/golden/make_distill_golden.py

utils/dataset_utils.py reads PLY files with ``plyfile``; where that is not installed a stand-in backed by
``io_formats.read_vertex_ply`` supplies ``PlyData.read``, and the reference's own ``load_gaussian_ply`` still picks
and orders the columns.  Inputs are regenerated from the seeds by the tests (``elastic_input``, ``vox_input``,
``write_scene``); only outputs are stored: SHA-256 digests of the returned arrays and the drawn noise grid sizes.
``random`` and ``np.random`` are both seeded with the case's seed right before the call."""
import collections.abc
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
from make_raster_golden import digest  # noqa: E402

from semantic_gaussians_b200.io_formats import gaussian_attribute_names, read_vertex_ply, write_vertex_ply  # noqa: E402

ELASTIC_PARAMS = ((0.2, 0.4), (0.8, 1.6))     # FeatureDataset.ELASTIC_DISTORT_PARAMS
SCALE_BOUND = (0.9, 1.1)
ROTATION_BOUND = ((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi))

# ElasticDistortion(ELASTIC_PARAMS)(xyz) alone: name -> (seed, P, cloud, dtype)
ELASTIC_CASES = {
    "elastic_f32": (10, 20000, "room", np.float32),
    "elastic_f64": (11, 20000, "room", np.float64),
    "elastic_thin": (12, 5000, "thin", np.float32),
    "elastic_single": (13, 1, "room", np.float32),
    "elastic_skip": (15, 2000, "room", np.float32),   # random.random() >= 0.95 right after seeding: no pass runs
}
# Voxelizer(0.02, augmentation with the dataset's bounds).voxelize on a float64 cloud: name -> (seed, P)
VOX_CASES = {"vox_f64": (20, 20000)}
# FeatureDataset(aug).__getitem__(0): name -> (seed, P, cloud, feature_type, aug)
DATASET_CASES = {
    "ds_all": (30, 20000, "room", "all", True),
    "ds_color": (31, 20000, "room", "color", True),
    "ds_thin": (32, 5000, "thin", "all", True),
    "ds_single": (33, 1, "room", "all", True),
    "ds_skip": (15, 5000, "room", "all", True),       # the distortion gate skips
    "ds_noaug": (35, 5000, "room", "all", False),
}
FEATURE_C = 16
VOXEL_SIZE = 0.02


def cloud(rng, P, kind):
    """(P,3) float64 points of a scanned 6 x 5 x 3 m room, partly on floor and ceiling; ``thin`` is flat in z."""
    xyz = rng.uniform((0, 0, 0), (6, 5, 3), (P, 3))
    xyz[: P // 2, 2] = rng.choice([0.0, 2.95], P // 2)
    if kind == "thin":
        xyz[:, 2] = 1.25
    return xyz


def elastic_input(case):
    seed, P, kind, dtype = ELASTIC_CASES[case]
    return cloud(np.random.default_rng(seed + 500), P, kind).astype(dtype)


def vox_input(case):
    """(xyz (P,3) float64 not representable in float32, feats (P,56) float32)."""
    seed, P = VOX_CASES[case]
    rng = np.random.default_rng(seed + 500)
    return cloud(rng, P, "room") + rng.uniform(-1e-9, 1e-9, (P, 3)), rng.standard_normal((P, 56)).astype(np.float32)


def write_scene(case, root):
    """Writes one scene (degree-3 Gaussian PLY and fused-feature .pt) under ``root``; returns
    (gaussians_dir, point_dir) for FeatureDataset."""
    seed, P, kind, _, _ = DATASET_CASES[case]
    rng = np.random.default_rng(seed + 700)
    names = gaussian_attribute_names(3, 45)
    table = rng.standard_normal((P, len(names))).astype(np.float32)
    table[:, :3] = cloud(rng, P, kind)
    ply = os.path.join(root, "gaussians", "scene0", "point_cloud", "iteration_30000", "point_cloud.ply")
    write_vertex_ply(ply, names, table)
    mask = rng.random(P) < 0.6
    mask[0] = True
    feat = rng.standard_normal((int(mask.sum()), FEATURE_C)).astype(np.float16)
    feat[::7] = 0                          # all-zero target rows
    os.makedirs(os.path.join(root, "points", "scene0"))
    torch.save({"feat": torch.from_numpy(feat), "mask_full": torch.from_numpy(mask)},
               os.path.join(root, "points", "scene0", "feat_0.pt"))
    return os.path.join(root, "gaussians"), os.path.join(root, "points")


def seed_all(seed):
    random.seed(seed)
    np.random.seed(seed)


class record_noise_dims:
    """Context manager listing the shapes of the ``np.random.randn(*noise_dim, 3)`` draws made inside it."""

    def __enter__(self):
        self.dims, self._randn = [], np.random.randn

        def randn(*shape):
            self.dims.append(shape[:3])
            return self._randn(*shape)
        np.random.randn = randn
        return self

    def __exit__(self, *exc):
        np.random.randn = self._randn

    def array(self):
        return np.asarray(self.dims, np.int64).reshape(-1, 3)


def _plyfile_standin():
    class Prop:
        def __init__(self, name):
            self.name = name

    class Element:
        def __init__(self, cols):
            self._cols = cols
            self.properties = [Prop(n) for n in cols]

        def __getitem__(self, k):
            return self._cols[k]

    class PlyData:
        @staticmethod
        def read(path):
            return types.SimpleNamespace(elements=[Element(read_vertex_ply(path))])

    return types.SimpleNamespace(PlyData=PlyData, PlyElement=None)


def reference_modules():
    """(dataset.augmentation, dataset.fusion_utils, dataset.feature_dataset) of the reference tree."""
    collections.Sequence = collections.abc.Sequence      # fusion_utils.py uses the pre-3.10 names
    collections.Iterable = collections.abc.Iterable
    try:
        import plyfile  # noqa: F401
    except ImportError:
        sys.modules["plyfile"] = _plyfile_standin()
    sys.path.insert(0, REF)
    try:
        import importlib
        return tuple(importlib.import_module(f"dataset.{m}") for m in ("augmentation", "fusion_utils",
                                                                       "feature_dataset"))
    finally:
        sys.path.remove(REF)


def main():
    aug, fu, fd = reference_modules()
    out = {}
    for case, (seed, *_r) in ELASTIC_CASES.items():
        xyz = elastic_input(case)
        seed_all(seed)
        with record_noise_dims() as rec:
            got = aug.ElasticDistortion(ELASTIC_PARAMS)(xyz)
        out[f"{case}_xyz.sha256"] = digest(got)
        out[f"{case}_noise_dims"] = rec.array()
        print(case, got.dtype, rec.dims)
    for case, (seed, _) in VOX_CASES.items():
        xyz, feats = vox_input(case)
        vox = fu.Voxelizer(voxel_size=VOXEL_SIZE, use_augmentation=True, scale_augmentation_bound=SCALE_BOUND,
                           rotation_augmentation_bound=ROTATION_BOUND)
        seed_all(seed)
        coords, f, _, inverse, inds = vox.voxelize(xyz, feats, None, return_ind=True)
        out[f"{case}_coords.sha256"], out[f"{case}_feats.sha256"] = digest(coords), digest(f)
        out[f"{case}_inds"], out[f"{case}_inverse"] = inds.astype(np.int32), inverse.astype(np.int32)
        print(case, "M", len(inds))
    for case, (seed, _, _, feature_type, use_aug) in DATASET_CASES.items():
        with tempfile.TemporaryDirectory() as root:
            gdir, pdir = write_scene(case, root)
            ds = fd.FeatureDataset(gdir, pdir, 30000, VOXEL_SIZE, use_aug, feature_type)
            seed_all(seed)
            with record_noise_dims() as rec:
                locs, features, features_gt, mask, head_id = ds[0]
        for name, t in (("locs", locs), ("features", features), ("features_gt", features_gt), ("mask", mask)):
            out[f"{case}_{name}.sha256"] = digest(t.numpy())
        out[f"{case}_noise_dims"] = rec.array()
        print(case, "M", len(locs), "masked", int(mask.sum()), rec.dims, locs.dtype, features.dtype,
              features_gt.dtype, mask.dtype)
    path = os.path.join(HERE, "distill_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
