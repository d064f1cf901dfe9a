"""Measures the BASELINE.json configs K1..K5 on one GPU and prints a markdown table
(ours vs the compiled reference CUDA path vs the CPU pieces)."""
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from oracle import fusion_oracle as fo
from oracle import oracle as orc
from oracle import ref as refmod
from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200.fusion import PointCloudToImageMapper, normalize_fused
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras, room_cameras
from util import dev_cam, dev_scene, run_ours

dev = torch.device("cuda:0")
rows = []


def ev(fn, n, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def raster(name, P, W, H, C, use_features, want_depth, backward, kind="blob", refname=None, ref_bwd=None, reps=10,
           views=1):
    scene = make_scene(P, 0, kind=kind, sh=not use_features, channels=C if use_features else 0)
    cams = (orbit_cameras if kind == "blob" else room_cameras)(8, W, H)
    sc = dev_scene(scene, dev, requires_grad=backward)
    cms = [dev_cam(c, dev) for c in cams]
    bg = torch.zeros(C, device=dev)
    dL = torch.randn((C, H, W), device=dev) / (H * W) if backward else None
    it = [0]

    def ours():
        o = run_ours("rgbd" if want_depth else "chn", sc, cms[it[0] % 8], bg, use_features=use_features)
        it[0] += 1
        if backward:
            o["color"].backward(dL)
            for v in sc.values():
                if v is not None:
                    v.grad = None
        return o
    o = ours()
    P_vis = int((o["radii"] > 0).sum())
    t = ev(ours, reps)
    ref_ms = ref_b = None
    sd = {k: (v.detach() if v is not None else None) for k, v in sc.items()}
    cm = cms[1]
    kw = dict(bg=bg, means3D=sd["means3D"], opacities=sd["opacities"], viewmatrix=cm["viewmatrix"],
              projmatrix=cm["projmatrix"], campos=cm["campos"], tanfovx=cm["tanfovx"], tanfovy=cm["tanfovy"], W=W, H=H,
              shs=None if use_features else sd["shs"], colors_precomp=sd["features"] if use_features else None,
              scales=sd["scales"], rotations=sd["rotations"], num_channels=C)
    R = None
    if refname and refmod.available(refname):
        r = refmod.RefRasterizer(refname)
        R = r.forward(**kw)["R"]
        ref_ms = ev(lambda: r.forward(**kw), max(2, reps // 4), 1)
    if backward and ref_bwd and refmod.available(ref_bwd):
        r2 = refmod.RefRasterizer(ref_bwd)
        r2.forward(**kw)
        ref_b = ev(lambda: r2.backward(dL), 1, 1)
    rows.append(f"| {name} | {P} | {C} | {W}x{H} | {'fwd+bwd' if backward else 'fwd'} | {P_vis} | {R} | **{t:.3f}** | "
                f"{1e3 / t:.1f} | {'%.2f' % ref_ms if ref_ms else '—'}{(' + %.1f' % ref_b) if ref_b else ''} |")
    print(rows[-1], flush=True)
    del sc, scene
    torch.cuda.empty_cache()


def cpu_k1():
    scene = make_scene(10000, 0, sh=True)
    cam = orbit_cameras(1, 256, 256)[0]
    t0 = time.perf_counter()
    f = orc.forward(orc.scene_dict(scene), orc.cam_dict(cam), 256, 256, np.zeros(3, np.float32), want_depth=True)
    t1 = time.perf_counter()
    orc.backward(f, orc.scene_dict(scene), orc.cam_dict(cam), 256, 256, np.zeros(3, np.float32),
                 np.ones((3, 256, 256), np.float32))
    t2 = time.perf_counter()
    print(f"K1 CPU oracle ({orc.num_threads()} threads): fwd {1e3 * (t1 - t0):.1f} ms, bwd {1e3 * (t2 - t1):.1f} ms", flush=True)
    rows.append(f"| K1 CPU port ({orc.num_threads()} threads) | 10000 | 3 | 256x256 | fwd / bwd | | | {1e3 * (t1 - t0):.1f} / {1e3 * (t2 - t1):.1f} | | |")


def fusion_k5(P=2_000_000, C=512, w=640, h=480, nviews=6):
    scene = make_scene(P, 0, kind="room")
    cams = room_cameras(nviews, w, h)
    rng = np.random.default_rng(0)
    fm = torch.from_numpy(rng.standard_normal((C, h, w)).astype(np.float16)).to(dev)
    xyz = torch.as_tensor(scene.xyz, device=dev)
    fs = torch.zeros((P, C), device=dev)
    cnt = torch.zeros(P, device=dev)
    depth = torch.full((h, w), 2.5, device=dev)
    ctx = _lib.ctx_for(0, torch.cuda.current_stream(dev).cuda_stream)
    mappers = [PointCloudToImageMapper([w, h], 0.5, 10, c.intrinsics(), device=dev) for c in cams]
    k = [0]

    def one():
        i = k[0] % nviews
        k[0] += 1
        mappers[i].accumulate(cams[i].world_view_transform, xyz, fm, fs, cnt, depth)
    one()
    torch.cuda.synchronize()
    _lib.profile_enable(ctx, True)
    t = ev(one, nviews, 0)
    st = _lib.profile_read(ctx)
    _lib.profile_enable(ctx, False)
    nvis = int((cnt > 0).sum())
    # CPU reference pieces: numpy compute_mapping (single thread) + torch gather/accumulate, one view
    K = fo.rescale_intrinsics(cams[0].intrinsics(), [w, h])
    t0 = time.perf_counter()
    m = fo.compute_mapping(cams[0].world_view_transform, scene.xyz, [w, h], K, 0.5, 10, depth.cpu().numpy())
    t1 = time.perf_counter()
    fmc = fm.cpu()
    mt = torch.from_numpy(m)
    t2 = time.perf_counter()
    g = fmc[:, mt[:, 0], mt[:, 1]].permute(1, 0)
    fsc = torch.zeros((P, C))
    mk = mt[:, 2] != 0
    fsc[mk] += g[mk]
    t3 = time.perf_counter()
    stages = " ".join(f"{a}={v[0] / max(v[1], 1):.3f}" for a, v in st.items() if v[1])
    print(f"K5 fusion: {t:.3f} ms/view on GPU ({stages}); CPU: mapping {1e3 * (t1 - t0):.0f} ms + gather/accumulate "
          f"{1e3 * (t3 - t2):.0f} ms per view; visible-any {nvis}", flush=True)
    rows.append(f"| K5 fusion (per view) | {P} | {C} fp16 | {w}x{h} | project+gather+accumulate | {nvis} | | **{t:.3f}** | "
                f"{1e3 / t:.1f} | CPU numpy+torch: {1e3 * (t1 - t0 + t3 - t2):.0f} |")


if __name__ == "__main__":
    print(torch.cuda.get_device_name(0), "host threads", os.cpu_count(), flush=True)
    cpu_k1()
    raster("K1", 10000, 256, 256, 3, False, True, True, refname="rgbd", ref_bwd="rgbd", reps=20)
    raster("K2", 1_000_000, 1920, 1080, 3, False, True, False, refname="rgbd", reps=20)
    raster("K2 (+bwd)", 1_000_000, 1920, 1080, 3, False, True, True, refname="rgbd", ref_bwd="rgbd", reps=10)
    raster("K3 fwd", 1_000_000, 1920, 1080, 256, True, False, False, refname="chn", reps=10)
    raster("K3", 1_000_000, 1920, 1080, 256, True, False, True, refname="chn", ref_bwd="chn_c256", reps=10)
    raster("K4 (1 view, 1 GPU)", 3_000_000, 1296, 968, 512, True, False, True, kind="room", refname="chn", reps=4)
    fusion_k5()
    print("\n| config | P | C | WxH | pass | P_vis | R | ours ms/view | views/s | reference CUDA ms (fwd [+ bwd]) |\n|---|---|---|---|---|---|---|---|---|---|")
    print("\n".join(rows))
