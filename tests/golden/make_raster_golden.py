"""Generates tests/golden/raster_golden_k1.npz by running the UNMODIFIED compiled reference rasterizer
(oracle/_ref/libref_{rgbd,chn,chn_c100}.so, built by oracle/build.py) on the seeded K1-size scene (10k Gaussians,
256x256) and a 100-channel feature scene, on a GPU:

    python tests/golden/make_raster_golden.py

Inputs are regenerated from the seed by the tests; the file stores the reference's outputs and the opaque-state
fields the tests read.  To stay small, the largest arrays are stored as the SHA-256 of their bytes (for bit-exact
checks) plus a fixed seeded sample of entries and the array's max |x| (for tolerance checks): see SAMPLED."""
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

KEEP = ("k1_R", "k1_depth", "k1_radii", "k1_depths", "k1_means2D", "k1_conic_opacity", "k1_rgb", "k1_tiles_touched",
        "k1_point_list", "k1_n_contrib", "kf_R", "kf_radii", "kf_dL_dmeans3D")
SAMPLED = ("k1_color", "k1_dL_dsh", "k1_dL_dmeans2D", "k1_dL_dopacity", "k1_dL_dmeans3D", "k1_dL_dscales",
           "k1_dL_drotations", "kf_color", "kf_dL_dcolors")
K1 = dict(P=10000, W=256, H=256, seed=0)
KF = dict(P=3000, W=64, H=48, C=100, seed=11)        # feature raster (chn / chn_c100)


def golden_inputs(kind):
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    if kind == "k1":
        scene = make_scene(K1["P"], K1["seed"], sh=True)
        cam = orbit_cameras(1, K1["W"], K1["H"])[0]
        rng = np.random.default_rng(5)
        dL = rng.standard_normal((3, K1["H"], K1["W"])).astype(np.float32)
        bg = np.array([0.1, 0.2, 0.3], np.float32)
    else:
        scene = make_scene(KF["P"], KF["seed"], channels=KF["C"], scale_mean=0.04)
        cam = orbit_cameras(3, KF["W"], KF["H"])[1]
        rng = np.random.default_rng(6)
        dL = rng.standard_normal((KF["C"], KF["H"], KF["W"])).astype(np.float32)
        bg = (0.01 * np.arange(KF["C"])).astype(np.float32)
    return scene, cam, dL, bg


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(str((a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def shrink(full):
    out = {k: full[k] for k in KEEP}
    for k in SAMPLED:
        a = full[k]
        idx = np.unique(np.random.default_rng(sum(map(ord, k))).integers(0, a.size, 8192)).astype(np.int64)
        out.update({k + ".sha256": digest(a), k + ".idx": idx, k + ".sample": a.reshape(-1)[idx],
                    k + ".maxabs": np.float64(np.abs(a).max()), k + ".shape": np.array(a.shape, np.int64)})
    return out


def sample_pair(gold, key, ours):
    """(ours, reference) at the stored sample of a SAMPLED array, as float64, and the reference's max |x|."""
    a = np.asarray(ours, np.float64).reshape(-1)
    assert a.size == int(np.prod(gold[key + ".shape"])), key
    return a[gold[key + ".idx"]], gold[key + ".sample"].astype(np.float64), float(gold[key + ".maxabs"])


def frac_bad_sampled(gold, key, ours, rtol, atol_scale):
    a, b, m = sample_pair(gold, key, ours)
    return float((np.abs(a - b) > rtol * np.abs(b) + atol_scale * m).mean())


def main():
    from oracle import ref as refmod
    from util import dev_cam, dev_scene
    dev = torch.device("cuda:0")
    out = {}
    # ---- K1: RGB (SH degree 3) + median depth through the rgbd library, fwd + bwd
    scene, cam, dL, bg = golden_inputs("k1")
    sc, cm = dev_scene(scene, dev), dev_cam(cam, dev)
    r = refmod.RefRasterizer("rgbd")
    f = r.forward(bg=torch.as_tensor(bg, device=dev), means3D=sc["means3D"], opacities=sc["opacities"],
                  viewmatrix=cm["viewmatrix"], projmatrix=cm["projmatrix"], campos=cm["campos"],
                  tanfovx=cm["tanfovx"], tanfovy=cm["tanfovy"], W=cm["W"], H=cm["H"], shs=sc["shs"],
                  scales=sc["scales"], rotations=sc["rotations"], num_channels=3)
    out["k1_R"] = np.int64(f["R"])
    out["k1_color"] = f["color"].cpu().numpy()
    out["k1_depth"] = f["depth"].cpu().numpy()
    out["k1_radii"] = f["radii"].cpu().numpy()
    for name in ("depths", "means2D", "conic_opacity", "cov3D", "rgb", "clamped", "tiles_touched", "point_list",
                 "ranges", "n_contrib", "accum_alpha"):
        out["k1_" + name] = r.field(name).cpu().numpy()
    g = r.backward(torch.as_tensor(dL, device=dev))
    for k, v in g.items():
        out["k1_" + k] = v.cpu().numpy()
    # ---- KF: 100-channel feature raster; forward by the stock chn library, backward by the
    #      NUM_CHANNELS=100 rebuild (the stock backward is 3-channel only)
    scene, cam, dL, bg = golden_inputs("kf")
    sc, cm = dev_scene(scene, dev), dev_cam(cam, dev)
    kw = dict(bg=torch.as_tensor(bg, device=dev), means3D=sc["means3D"], opacities=sc["opacities"],
              viewmatrix=cm["viewmatrix"], projmatrix=cm["projmatrix"], campos=cm["campos"], tanfovx=cm["tanfovx"],
              tanfovy=cm["tanfovy"], W=cm["W"], H=cm["H"], colors_precomp=sc["features"], scales=sc["scales"],
              rotations=sc["rotations"], num_channels=KF["C"])
    r0 = refmod.RefRasterizer("chn")
    f0 = r0.forward(**kw)
    out["kf_R"] = np.int64(f0["R"])
    out["kf_color"] = f0["color"].cpu().numpy()
    out["kf_radii"] = f0["radii"].cpu().numpy()
    out["kf_n_contrib"] = r0.field("n_contrib").cpu().numpy()
    out["kf_accum_alpha"] = r0.field("accum_alpha").cpu().numpy()
    out["kf_point_list"] = r0.field("point_list").cpu().numpy()
    r1 = refmod.RefRasterizer("chn_c100")
    r1.forward(**kw)
    g = r1.backward(torch.as_tensor(dL, device=dev))
    for k, v in g.items():
        if k != "dL_dsh":
            out["kf_" + k] = v.cpu().numpy()
    path = os.path.join(ROOT, "tests", "golden", "raster_golden_k1.npz")
    np.savez_compressed(path, **shrink(out))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
