"""Lifting feature maps onto the Gaussians by their blend weights (sgb_lift_batch, fusion.lift_views / lift_scene) on
the GPU: against the float64 restatement (lift_ref.lift) on the kernels' own per-Gaussian state and tile lists at
every channel count, map dtype, image width and map alignment the dL/dfeature contraction branches on; against the
autograd route it replaces; and the invariants a user relies on.

Which case reaches which branch of dfeature_persistent_kernel<T>:
  C = 1 .. 512, fp16 / fp32 ...... 64-channel items, partial last item, red16 on and off (C % 4)
  w164 ........................... W % 8 = 4: fp32 by TMA, fp16 staged with plain loads
  w161 ........................... W % 4 = 1: both staged (cp.async for fp32, plain loads for fp16), partial tiles
  map_offset ..................... map base 4 (fp32) / 2 (fp16) bytes off 16-byte alignment: staged
  sparse, dense_faint ............ empty tiles; lists past the first weight-pool guess (overflow and retry)"""
import ctypes as Ct
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blend_ref as br  # noqa: E402
import lift_ref as lr  # noqa: E402
from raster_check import read_state  # noqa: E402
from util import dev_cam, dev_scene  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.scene_synth import look_at_camera, make_scene, orbit_cameras  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F16, F32 = torch.float16, torch.float32


def _placed(t, offset_bytes):
    """A copy of t whose data pointer is offset_bytes past a 16-byte boundary."""
    es = t.element_size()
    buf = torch.zeros(t.numel() + 16 // es, dtype=t.dtype, device=t.device)
    v = buf[offset_bytes // es: offset_bytes // es + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == offset_bytes
    return v


def _native(sc, cams, W, H, Cn, antialiasing=False):
    """(ViewInputs of the Gaussians without colours, sgb_camera array, the tensors they point into)."""
    cms = [dev_cam(c, DEV) for c in cams]
    inp = _lib.ViewInputs(P=sc["means3D"].shape[0], D=0, M=0, W=W, H=H, C=Cn, background=None,
                          means3D=sc["means3D"].data_ptr(), shs=None, colors_precomp=None,
                          opacities=sc["opacities"].data_ptr(), scales=sc["scales"].data_ptr(), scale_modifier=1.0,
                          rotations=sc["rotations"].data_ptr(), cov3D_precomp=None, viewmatrix=None, projmatrix=None,
                          campos=None, tan_fovx=0.0, tan_fovy=0.0, prefiltered=0, debug=0,
                          antialiasing=int(bool(antialiasing)))
    cam_arr = (_lib.Camera * len(cams))(*[_lib.Camera(c["viewmatrix"].data_ptr(), c["projmatrix"].data_ptr(),
                                                      c["campos"].data_ptr(), c["tanfovx"], c["tanfovy"]) for c in cms])
    return inp, cam_arr, cms


def forward_states(sc, cams, W, H, antialiasing=False):
    """Every view's kernel state (means2D, conic_opacity, point_list, ranges, final_T) from C = 8 forwards of at most
    8 views on a fresh ctx; None for a view without instances."""
    if len(cams) > _lib.MAX_BATCH:
        return [st for lo in range(0, len(cams), _lib.MAX_BATCH)
                for st in forward_states(sc, cams[lo:lo + _lib.MAX_BATCH], W, H, antialiasing)]
    lib = _lib.load()
    V, P = len(cams), sc["means3D"].shape[0]
    inp, cam_arr, keep = _native(sc, cams, W, H, 8, antialiasing)
    feats, bg = torch.zeros((P, 8), device=DEV), torch.zeros(8, device=DEV)
    inp.colors_precomp, inp.background = feats.data_ptr(), bg.data_ptr()
    ptrs = lambda ts: (Ct.c_void_p * V)(*[t.data_ptr() for t in ts])
    u8 = dict(dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    ctx = Ct.c_void_p()
    _lib.check(lib.sgb_ctx_create(Ct.byref(ctx), 0), "sgb_ctx_create")
    try:
        radii = [torch.empty((P,), dtype=torch.int32, device=DEV) for _ in cams]
        geom = [torch.empty((lib.sgb_geometry_bytes(P),), **u8) for _ in cams]
        img = [torch.empty((lib.sgb_image_bytes(W, H),), **u8) for _ in cams]
        Rs = (Ct.c_int64 * V)()
        _lib.check(lib.sgb_forward_geometry_batch(ctx, Ct.byref(inp), V, cam_arr, ptrs(geom), ptrs(radii), Rs, stream),
                   "geometry")
        binning = [torch.empty((lib.sgb_binning_bytes(R),), **u8) for R in Rs]
        color = [torch.empty((8, H, W), device=DEV) for _ in cams]
        _lib.check(lib.sgb_forward_render_batch(ctx, Ct.byref(inp), V, cam_arr, Rs, ptrs(geom), ptrs(binning),
                                                ptrs(img), ptrs(radii), ptrs(color), None, stream), "render")
        return [read_state(lib, P, Rs[v], W, H, geom[v], binning[v], img[v]) if Rs[v] else None for v in range(V)]
    finally:
        torch.cuda.synchronize(DEV)
        lib.sgb_ctx_destroy(ctx)


def lift_native(sc, cams, W, H, maps, ctx=None, antialiasing=False):
    """sgb_lift_batch of len(cams) views (maps: (C, H, W) tensors of one dtype) on a fresh ctx or the one given.
    Returns (feat_sum, weight_sum, weight-pool chunks of the last view)."""
    lib = _lib.load()
    V, P, Cn = len(cams), sc["means3D"].shape[0], maps[0].shape[0]
    inp, cam_arr, keep = _native(sc, cams, W, H, Cn, antialiasing)
    fs, ws = torch.zeros((P, Cn), device=DEV), torch.zeros(P, device=DEV)
    dt = _lib.FEAT_F16 if maps[0].dtype == F16 else _lib.FEAT_F32
    own = ctx is None
    if own:
        ctx = Ct.c_void_p()
        _lib.check(lib.sgb_ctx_create(Ct.byref(ctx), 0), "sgb_ctx_create")
    try:
        _lib.check(lib.sgb_lift_batch(ctx, Ct.byref(inp), V, cam_arr, (Ct.c_void_p * V)(*[m.data_ptr() for m in maps]),
                                      dt, fs.data_ptr(), ws.data_ptr(), torch.cuda.current_stream(DEV).cuda_stream),
                   "sgb_lift_batch")
        torch.cuda.synchronize(DEV)
        chunks = lib.sgb_ctx_view_stat(ctx, 1)
    finally:
        if own:
            lib.sgb_ctx_destroy(ctx)
    return fs, ws, chunks


def check_lift(scene, cams, Cn, dtype, *, map_offset=0, seed=0, antialiasing=False):
    """Lift random maps (zero at each view's fragile pixels) of len(cams) views natively and compare feat_sum and
    weight_sum with the sum of the views' float64 restatements (on the kernels' state: with antialiasing the
    record's opacity is o h).  Returns the errors and statistics."""
    W, H = cams[0].image_width, cams[0].image_height
    sc = dev_scene(scene, DEV)
    states = forward_states(sc, cams, W, H, antialiasing)
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = scene.P
    want_f = torch.zeros((P, Cn), dtype=torch.float64, device=DEV)
    want_w = torch.zeros(P, dtype=torch.float64, device=DEV)
    ok = torch.ones(P, dtype=torch.bool, device=DEV)
    maps, frag, lens = [], [], []
    for st in states:
        m = torch.randn((Cn, H * W), device=DEV, generator=g)
        if st is not None:
            frag_v = lr.lift(st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], m.reshape(Cn, H, W),
                             W, H)["fragile"]
            m[:, frag_v] = 0.0
        m = m.reshape(Cn, H, W).to(dtype)
        if st is not None:
            r = lr.lift(st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], m, W, H)
            want_f += r["feat_sum"]
            want_w += r["weight_sum"]
            ok &= r["weight_ok"]
            frag.append(float(r["fragile"].double().mean()))
            rg = st["ranges"].long()
            lens.append(rg[:, 1] - rg[:, 0])
        maps.append(_placed(m, map_offset))
    fs, ws, chunks = lift_native(sc, cams, W, H, maps, antialiasing=antialiasing)
    seen = want_w > 0
    assert int(seen.sum()) > 0 and int((ok & seen).sum()) > 0
    errs = dict(feat_sum=br.compare(fs, want_f), weight_sum=br.compare(ws[ok], want_w[ok]))
    return dict(errs=errs, fragile=max(frag, default=0.0), chunks=chunks, fs=fs, ws=ws, states=states, maps=maps,
                lens=torch.cat(lens).cpu() if lens else torch.zeros(0))


def _assert_ok(res):
    assert res["fragile"] <= 0.02, res["fragile"]
    assert all(v <= 1.0 for v in res["errs"].values()), res["errs"]


CASES = {f"c{C}_{'f16' if dt is F16 else 'f32'}": (20000, 160, 96, C, dt, 0.02, None, 0)
         for C in (1, 3, 5, 63, 64, 65, 257, 512) for dt in (F16, F32)}
CASES.update({
    "w164_f16": (20000, 164, 96, 64, F16, 0.02, None, 0),
    "w164_f32": (20000, 164, 96, 64, F32, 0.02, None, 0),
    "w161_h100_f16": (20000, 161, 100, 33, F16, 0.02, None, 0),
    "w161_h100_f32": (20000, 161, 100, 33, F32, 0.02, None, 0),
    "map_offset_f16": (20000, 160, 96, 64, F16, 0.02, None, 2),
    "map_offset_f32": (20000, 160, 96, 64, F32, 0.02, None, 4),
    "tile_13x7_f16": (20000, 13, 7, 16, F16, 0.02, None, 0),
    "sparse_f16": (60, 160, 96, 32, F16, 0.02, None, 0),
    "dense_faint_f16": (100000, 128, 96, 65, F16, 0.05, 0.02, 0),
})


@pytest.mark.parametrize("name", list(CASES))
def test_lift_matches_fp64(name):
    P, W, H, Cn, dt, scale, opacity, off = CASES[name]
    scene = make_scene(P, seed=50, channels=1, scale_mean=scale)
    if opacity is not None:
        scene.opacity[:] = opacity
    res = check_lift(scene, [orbit_cameras(4, W, H)[1]], Cn, dt, map_offset=off)
    print(f"\n[lift fp64] {name}: fragile={res['fragile']:.4%} " +
          " ".join(f"{k}={v:.3g}" for k, v in res["errs"].items()))
    _assert_ok(res)
    L = res["lens"]
    if name.startswith("sparse"):
        assert int((L == 0).sum()) > 0
    if name.startswith("dense_faint"):
        assert res["chunks"] > L.numel() * 8   # the first guess of 8 chunks per tile overflowed and was retried


@pytest.mark.parametrize("V,dt", [(3, F16), (8, F32)])
def test_batched_lift_matches_fp64(V, dt):
    scene = make_scene(20000, seed=51, channels=1)
    cams = orbit_cameras(V, 160, 96)
    if V == 3:   # a middle view that looks away from the scene: R = 0
        cams[1] = look_at_camera((3.0, 0.0, 0.4), (6.0, 0.0, 0.4), 160, 96)
    res = check_lift(scene, cams, 65, dt, seed=V)
    if V == 3:
        assert res["states"][1] is None
    _assert_ok(res)


# ---- the Python path ------------------------------------------------------------------------------------------

class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


class View:
    def __init__(self, c):
        self.image_width, self.image_height, self.FoVx, self.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
        self.world_view_transform = torch.as_tensor(c.world_view_transform, device=DEV)
        self.full_proj_transform = torch.as_tensor(c.full_proj_transform, device=DEV)
        self.camera_center = torch.as_tensor(c.camera_center, device=DEV)
        self.intrinsics = c.intrinsics()


def _model(P, seed, **kw):
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    scene = make_scene(P, seed, sh=True, **kw)
    return GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, shs=scene.shs,
                                        device=DEV)


def _model_inputs(pc):
    """The Gaussian-side tensors render_chn_batch / lift_views hand to the native calls."""
    with torch.no_grad():
        return dict(means3D=pc.get_xyz.contiguous(), opacities=pc.get_opacity.contiguous(),
                    scales=pc.get_scaling.contiguous(), rotations=pc.get_rotation.contiguous())


def test_lift_views_eleven_views_split_in_python_matches_fp64():
    from semantic_gaussians_b200.fusion import lift_views
    pc = _model(20000, 52)
    W, H, Cn = 96, 64, 40
    cams = orbit_cameras(11, W, H)
    cams[4] = look_at_camera((3.0, 0.0, 0.4), (6.0, 0.0, 0.4), W, H)   # R = 0
    views = [View(c) for c in cams]
    sc = _model_inputs(pc)
    states = forward_states(sc, cams, W, H)
    assert states[4] is None
    g = torch.Generator(device=DEV).manual_seed(9)
    maps, want_f, want_w, ok = [], 0, 0, torch.ones(20000, dtype=torch.bool, device=DEV)
    for st in states:
        m = torch.randn((Cn, H, W), device=DEV, generator=g).half()
        if st is not None:
            r = lr.lift(st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], m, W, H)
            m.reshape(Cn, -1)[:, r["fragile"]] = 0.0
            r = lr.lift(st["means2D"], st["conic_opacity"], st["point_list"], st["ranges"], m, W, H)
            want_f, want_w, ok = want_f + r["feat_sum"], want_w + r["weight_sum"], ok & r["weight_ok"]
        maps.append(m)
    fs, ws = torch.zeros((20000, Cn), device=DEV), torch.zeros((20000, 1), device=DEV)
    calls = []
    assert lift_views(pc, views, lambda i: calls.append(i) or maps[i], Pipe, fs, ws) == 11
    assert calls == list(range(11))
    assert br.compare(fs, want_f) <= 1.0
    assert br.compare(ws.view(-1)[ok], want_w[ok]) <= 1.0


def test_lift_views_mixed_map_dtypes_fetch_each_map_once():
    """A dtype change splits the native batch; the map fetched at the split is not fetched again."""
    from semantic_gaussians_b200.fusion import lift_views
    pc = _model(20000, 59)
    views = [View(c) for c in orbit_cameras(5, 96, 64)]
    g = torch.Generator(device=DEV).manual_seed(8)
    maps = [torch.randn((20, 64, 96), device=DEV, generator=g).half() for _ in views]
    mixed = [m if i in (0, 1, 3) else m.float() for i, m in enumerate(maps)]
    calls = []
    out = []
    for src in (maps, mixed):
        fs, ws = torch.zeros((20000, 20), device=DEV), torch.zeros(20000, device=DEV)
        calls.clear()
        lift_views(pc, views, lambda i: calls.append(i) or src[i], Pipe, fs, ws)
        assert calls == list(range(5))
        out.append((fs, ws))
    assert br.compare(out[1][0], out[0][0]) <= 1.0 and br.compare(out[1][1], out[0][1]) <= 1.0


def test_lift_equals_the_autograd_feature_gradient():
    """feat_sum of an fp32 map == features.grad of render_chn(...)["render"].backward(map): the same contraction
    on the same weights, summed in another order."""
    from semantic_gaussians_b200.fusion import lift_views
    from semantic_gaussians_b200.renderer import render_chn
    pc = _model(30000, 53)
    W, H, Cn = 200, 120, 96
    view = View(orbit_cameras(3, 320, 240)[0])
    F = torch.randn((Cn, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    feats = torch.zeros((30000, Cn), device=DEV, requires_grad=True)
    out = render_chn(view, pc, Pipe, torch.zeros(Cn, device=DEV), num_channels=Cn, override_color=feats,
                     override_shape=(W, H))
    out["render"].backward(F)
    fs, ws = torch.zeros((30000, Cn), device=DEV), torch.zeros(30000, device=DEV)
    lift_views(pc, [view], [F], Pipe, fs, ws)
    assert float(feats.grad.abs().max()) > 0
    assert br.compare(fs, feats.grad) <= 1.0


def test_weight_sums_add_up_to_the_rendered_opacity_and_constant_maps_lift_exactly():
    from semantic_gaussians_b200.fusion import lift_views, normalize_fused
    pc = _model(30000, 54)
    W, H = 160, 120
    cams = orbit_cameras(2, W, H)
    states = forward_states(_model_inputs(pc), cams, W, H)
    views = [View(c) for c in cams]
    c = torch.linspace(-2.0, 3.0, 7, device=DEV)
    for v in range(2):   # per view: sum_i weight_sum_i = sum_p (1 - final_T_p)
        fs, ws = torch.zeros((30000, 7), device=DEV), torch.zeros(30000, device=DEV)
        lift_views(pc, [views[v]], [c[:, None, None].expand(7, H, W).contiguous().half()], Pipe, fs, ws)
        total = float((1.0 - states[v]["final_T"].double()).sum())
        assert abs(float(ws.double().sum()) - total) <= 1e-5 * total, (float(ws.double().sum()), total)
        seen = ws > 0
        normalize_fused(fs, ws)
        want = c.half().float()[None, :].expand(int(seen.sum()), 7)
        assert torch.allclose(fs[seen], want, rtol=1e-5, atol=1e-6), float((fs[seen] - want).abs().max())
        assert float(fs[~seen].abs().max()) == 0.0 if bool((~seen).any()) else True


def test_fp16_map_equals_its_fp32_widening():
    from semantic_gaussians_b200.fusion import lift_views
    pc = _model(20000, 55)
    view = View(orbit_cameras(2, 168, 96)[1])   # W % 8 == 0: both dtypes by TMA
    m16 = torch.randn((130, 96, 168), device=DEV, generator=torch.Generator(device=DEV).manual_seed(4)).half()
    out = []
    for m in (m16, m16.float()):
        fs, ws = torch.zeros((20000, 130), device=DEV), torch.zeros(20000, device=DEV)
        lift_views(pc, [view], [m], Pipe, fs, ws)
        out.append((fs, ws))
    assert br.compare(out[0][0], out[1][0]) <= 1.0 and br.compare(out[0][1], out[1][1]) <= 1.0


def test_profiling_shows_no_blend_and_one_contraction_per_view():
    from semantic_gaussians_b200.fusion import lift_views
    pc = _model(20000, 56)
    views = [View(c) for c in orbit_cameras(3, 160, 96)]
    maps = [torch.randn((64, 96, 160), device=DEV).half() for _ in views]
    fs, ws = torch.zeros((20000, 64), device=DEV), torch.zeros(20000, device=DEV)
    lift_views(pc, views[:1], maps[:1], Pipe, fs, ws)   # warm-up
    ctx = _lib.ctx_for(0, torch.cuda.current_stream(DEV).cuda_stream)
    _lib.profile_enable(ctx, True)
    try:
        lift_views(pc, views, maps, Pipe, fs, ws)
        prof = _lib.profile_read(ctx)
    finally:
        _lib.profile_enable(ctx, False)
    assert prof["blend_fwd"][1] == 0 and prof["blend_bwd"][1] == 0 and prof["geom_bwd"][1] == 0
    assert prof["dfeature"][1] == 3 and prof["weight_sum"][1] == 3 and prof["alpha_pass"][1] >= 3


def test_lift_between_forward_and_backward_leaves_gradients_unchanged():
    """render_chn_batch (V = 8) -> lift_views -> backward on one ctx: the lift takes the forward's weight-pool slots,
    and the backward rebuilds them."""
    from semantic_gaussians_b200.fusion import lift_views
    from semantic_gaussians_b200.renderer import render_chn_batch
    pc = _model(20000, 57)
    W, H, Cn = 128, 96, 24
    views = [View(c) for c in orbit_cameras(8, W, H)]
    g = torch.Generator(device=DEV).manual_seed(5)
    dL = [torch.randn((Cn, H, W), device=DEV, generator=g) for _ in views]
    maps = [torch.randn((Cn, H, W), device=DEV, generator=g).half() for _ in views]
    base = torch.randn((20000, Cn), device=DEV, generator=g)

    def step(lift):
        pc._xyz.requires_grad_(True)
        pc._xyz.grad = None
        feats = base.clone().requires_grad_(True)
        outs = render_chn_batch(views, pc, Pipe, torch.zeros(Cn, device=DEV), num_channels=Cn, override_color=feats)
        if lift:
            lift_views(pc, views, maps, Pipe, torch.zeros((20000, Cn), device=DEV), torch.zeros(20000, device=DEV))
        sum((o["render"] * d).sum() for o, d in zip(outs, dL)).backward()
        return feats.grad.clone(), pc._xyz.grad.clone()

    want, got = step(False), step(True)
    pc._xyz.requires_grad_(False)
    assert br.compare(got[0], want[0]) <= 1.0
    assert br.compare(got[1], want[1]) <= 1.0


def test_lift_scene_output_and_sharded_path():
    from semantic_gaussians_b200.distributed import fuse_views_sharded
    from semantic_gaussians_b200.fusion import lift_scene, lift_views, normalize_fused
    from semantic_gaussians_b200.io_formats import save_fused_features
    pc = _model(20000, 58)
    W, H, Cn = 120, 90, 32
    cams = orbit_cameras(10, W, H)
    views = [View(c) for c in cams]
    g = torch.Generator(device=DEV).manual_seed(6)
    maps = [torch.randn((Cn, H, W), device=DEV, generator=g).half() for _ in views]
    pc.create_semantic(Cn)
    out = lift_scene(pc, views, maps, Pipe, every=3)
    assert set(out) == {"features", "mask", "views", "weights"} and out["views"] == 4
    assert out["features"].dtype == torch.float32 and out["features"].shape == (20000, Cn)
    assert out["mask"].dtype == torch.bool and out["mask"].shape == (20000,)
    assert out["weights"].dtype == torch.float32 and out["weights"].shape == (20000,)
    assert torch.equal(out["mask"], out["weights"] > 0)
    assert 0 < int(out["mask"].sum()) < 20000
    assert float(out["features"][~out["mask"]].abs().max()) == 0.0
    assert out["features"] is pc._features_semantic and torch.equal(pc._times.view(-1), out["weights"])
    # the same views through lift_views, and through the sharded loop with world = 1
    sel = [0, 3, 6, 9]
    fs, ws = torch.zeros((20000, Cn), device=DEV), torch.zeros(20000, device=DEV)
    lift_views(pc, [views[i] for i in sel], [maps[i] for i in sel], Pipe, fs, ws)
    mask = ws > 0
    normalize_fused(fs, ws)
    assert torch.equal(mask, out["mask"]) and br.compare(out["features"], fs) <= 1.0
    fs2, ws2 = torch.zeros((20000, Cn), device=DEV), torch.zeros(20000, device=DEV)
    fuse_views_sharded(len(sel), lambda k: lift_views(pc, [views[sel[k]]], [maps[sel[k]]], Pipe, fs2, ws2), fs2, ws2,
                       normalize_fused, rank=0, world=1)
    assert br.compare(fs2, fs) <= 1.0
    save_fused_features(os.devnull, out["features"][out["mask"]], out["mask"])
