"""Generates tests/golden/voxel_golden.npz by running the REFERENCE's own Voxelizer.voxelize (imported from
/root/reference/dataset/fusion_utils.py, with the collections.Sequence/Iterable aliases it needs on Python >= 3.10)
on seeded synthetic clouds.  Run in the build container:

    python tests/golden/make_voxel_golden.py

Inputs are regenerated from the seed by the tests (``voxel_inputs``); only outputs are stored, per case: the two
drawn matrices (``M_v``, ``M_r``), ``inds`` and ``inds_reconstruct`` (int32), and the SHA-256 of the returned
coords (float64) and feats (float32), which the tests compare bit for bit.  ``np.random`` is seeded with the case's
seed right before ``voxelize``, so an augmented case pins the reference's order of random draws."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_fusion_golden import import_reference_mapper  # noqa: E402
from make_raster_golden import digest  # noqa: E402

# dataset/feature_dataset.py:13-18: the augmentation a FeatureDataset(aug=True) voxelizes with
SCALE_BOUND = (0.9, 1.1)
ROTATION_BOUND = ((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi))

# name: (seed, P, cloud, voxel_size, augmentation)
CASES = {
    "plain_002": (0, 20000, "room", 0.02, False),
    "plain_005": (1, 20000, "room", 0.05, False),
    "aug_002": (2, 20000, "room", 0.02, True),
    "aug_005": (3, 20000, "blob", 0.05, True),
    "negative": (4, 20000, "negative", 0.02, False),
    "duplicates": (5, 20000, "duplicates", 0.02, False),
    "single": (6, 1, "room", 0.02, True),
}


def voxel_inputs(case):
    """(xyz (P,3) float32, feats (P,56) float32) of a case: the layout of get_locs_and_features("all")."""
    seed, P, cloud, _, _ = CASES[case]
    rng = np.random.default_rng(seed + 300)
    if cloud == "room":            # a scanned room: points spread over a few metres, partly on surfaces
        xyz = rng.uniform((0, 0, 0), (6, 5, 3), (P, 3))
        xyz[: P // 2, 2] = rng.choice([0.0, 2.95], P // 2)
    elif cloud == "blob":          # dense: many points per voxel
        xyz = rng.standard_normal((P, 3)) * 0.3 + 1.5
    elif cloud == "negative":      # every coordinate below zero
        xyz = rng.uniform((-7, -4, -3), (-0.5, -0.01, -1e-3), (P, 3))
    else:                          # exact duplicates of a quarter of the points, shuffled
        base = rng.uniform(-2, 2, (P // 4, 3))
        xyz = base[rng.permutation(np.arange(P) % (P // 4))]
    feats = rng.standard_normal((P, 56))
    return xyz.astype(np.float32), feats.astype(np.float32)


def reference_voxelizer_class():
    return sys.modules[import_reference_mapper().__module__].Voxelizer


def voxelizer_kwargs(case):
    _, _, _, voxel_size, aug = CASES[case]
    kw = dict(voxel_size=voxel_size)
    if aug:
        kw.update(use_augmentation=True, scale_augmentation_bound=SCALE_BOUND,
                  rotation_augmentation_bound=ROTATION_BOUND)
    return kw


def main():
    Voxelizer = reference_voxelizer_class()
    out = {}
    for case, (seed, *_rest) in CASES.items():
        xyz, feats = voxel_inputs(case)
        vox = Voxelizer(**voxelizer_kwargs(case))
        np.random.seed(seed)
        M_v, M_r = vox.get_transformation_matrix()
        np.random.seed(seed)
        coords, f, labels, inverse, inds = vox.voxelize(xyz, feats, None, return_ind=True)
        assert labels is None and coords.dtype == np.float64 and f.dtype == np.float32
        out[f"{case}_M_v"], out[f"{case}_M_r"] = M_v, M_r
        out[f"{case}_inds"] = np.asarray(inds).astype(np.int32)
        out[f"{case}_inds_reconstruct"] = np.asarray(inverse).astype(np.int32)
        out[f"{case}_coords.sha256"] = digest(coords)
        out[f"{case}_feats.sha256"] = digest(f)
        print(case, "P", len(xyz), "M", len(inds))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "voxel_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
