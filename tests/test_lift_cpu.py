"""Lifting feature maps onto the Gaussians by their blend weights, without a GPU: the float64 lift restatement
(lift_ref.lift) against a per-pixel loop and against the blend backward it is the feature gradient of, the
argument checks of lift_views / lift_scene and of sgb_lift_batch (refused before any ctx is used or anything is
enqueued), and what the built library contains."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blend_ref as br  # noqa: E402
import lift_ref as lr  # noqa: E402
from oracle import oracle as orc  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

E_INVALID = -1   # SGB_E_INVALID, include/sgb200.h


@pytest.fixture(scope="module")
def tiny():
    """A 37 x 21 view (partial tiles both ways) of 400 Gaussians: the oracle's preprocess and binning, a map."""
    P, W, H, Cn = 400, 37, 21, 3
    scene = make_scene(P, seed=12, channels=Cn, scale_mean=0.06)
    cam = orbit_cameras(4, W, H)[2]
    fo = orc.forward(orc.scene_dict(scene), orc.cam_dict(cam), W, H, np.zeros(Cn, np.float32), features=scene.features)
    pre, b = fo["pre"], fo["bin"]
    maps = np.random.default_rng(1).standard_normal((Cn, H, W))
    return dict(means2D=torch.from_numpy(pre["means2D"]), conic_opacity=torch.from_numpy(pre["conic_opacity"]),
                point_list=torch.from_numpy(b["point_list"].astype(np.int64)),
                ranges=torch.from_numpy(b["ranges"].astype(np.int64)), maps=torch.from_numpy(maps), W=W, H=H,
                features=torch.from_numpy(scene.features))


def _per_pixel_lift(st):
    """forward.cu's walk one pixel at a time in Python floats, accumulating w F and w per Gaussian."""
    W, H = st["W"], st["H"]
    mean, con = st["means2D"].double().numpy(), st["conic_opacity"].double().numpy()
    pl, rg, F = st["point_list"].numpy(), st["ranges"].numpy().reshape(-1, 2), st["maps"].numpy()
    P, Cn = mean.shape[0], F.shape[0]
    feat, wsum = np.zeros((P, Cn)), np.zeros(P)
    gx = (W + 15) // 16
    for y in range(H):
        for x in range(W):
            s, e = rg[(y // 16) * gx + x // 16]
            T = 1.0
            for g in pl[s:e]:
                dx, dy = mean[g, 0] - x, mean[g, 1] - y
                a, b, c, o = con[g]
                power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
                if power > 0:
                    continue
                alpha = min(br.ALPHA_MAX, o * math.exp(power))
                if alpha < br.ALPHA_MIN:
                    continue
                if T * (1 - alpha) < br.T_MIN:
                    break
                w = alpha * T
                feat[g] += w * F[:, y, x]
                wsum[g] += w
                T *= 1 - alpha
    return feat, wsum


def test_lift_restatement_matches_per_pixel_loop(tiny):
    got = lr.lift(tiny["means2D"], tiny["conic_opacity"], tiny["point_list"], tiny["ranges"], tiny["maps"],
                  tiny["W"], tiny["H"])
    feat, wsum = _per_pixel_lift(tiny)
    assert wsum.max() > 0 and (wsum > 0).sum() > 50
    np.testing.assert_allclose(got["weight_sum"].numpy(), wsum, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(got["feat_sum"].numpy(), feat, rtol=1e-12, atol=1e-12)


def test_lift_numerator_is_the_blend_backward_feature_gradient(tiny):
    st = {k: tiny[k] for k in ("means2D", "conic_opacity", "point_list", "ranges")}
    got = lr.lift(**st, maps=tiny["maps"], W=tiny["W"], H=tiny["H"])
    bwd = br.blend_backward(**st, features=tiny["features"], bg=torch.zeros(3), W=tiny["W"], H=tiny["H"],
                            dL_dpix=tiny["maps"])
    np.testing.assert_allclose(got["feat_sum"].numpy(), bwd["dL_dcolors"].numpy(), rtol=1e-12, atol=1e-12)


def test_constant_map_lifts_to_its_value(tiny):
    c = torch.full((3, tiny["H"], tiny["W"]), 0.75, dtype=torch.float64)
    got = lr.lift(tiny["means2D"], tiny["conic_opacity"], tiny["point_list"], tiny["ranges"], c, tiny["W"], tiny["H"])
    seen = got["weight_sum"] > 0
    mean = got["feat_sum"][seen] / got["weight_sum"][seen, None]
    assert torch.allclose(mean, torch.full_like(mean, 0.75), rtol=1e-12, atol=0)


# ---- argument checks ------------------------------------------------------------------------------------------

class _Gaussians:
    def __init__(self, P=5):
        self.get_xyz = torch.zeros(P, 3)


class _Pipe:
    compute_cov3d_python = False
    convert_shs_python = False
    debug = False


@pytest.mark.parametrize("make,exc,match", [
    (lambda: torch.zeros(4, 6, 8, dtype=torch.int32), TypeError, "float16 or float32"),
    (lambda: torch.zeros(4, 6, 8, dtype=torch.float64), TypeError, "float16 or float32"),
    (lambda: np.zeros((4, 6, 8), np.float32), TypeError, "torch.Tensor"),
    (lambda: torch.zeros(6, 8), ValueError, "must be"),
    (lambda: torch.zeros(3, 6, 8), ValueError, "C=4"),
])
def test_lift_views_rejects_bad_maps(make, exc, match):
    from semantic_gaussians_b200.fusion import lift_views
    with pytest.raises(exc, match=match):
        lift_views(_Gaussians(), [object()], [make()], _Pipe, torch.zeros(5, 4), torch.zeros(5))


def test_lift_views_rejects_mismatched_map_sizes():
    from semantic_gaussians_b200.fusion import lift_views
    maps = [torch.zeros(4, 6, 8), torch.zeros(4, 6, 8, dtype=torch.float16), torch.zeros(4, 6, 9)]
    with pytest.raises(ValueError, match="share the render size"):
        lift_views(_Gaussians(), [object()] * 3, maps, _Pipe, torch.zeros(5, 4), torch.zeros(5))


@pytest.mark.parametrize("fs,ws,exc", [
    (torch.zeros(5, 4, dtype=torch.float64), torch.zeros(5), TypeError),
    (torch.zeros(5, 4), torch.zeros(5, dtype=torch.float16), TypeError),
    (torch.zeros(6, 4), torch.zeros(5), ValueError),
    (torch.zeros(5, 4), torch.zeros(4), ValueError),
    (torch.zeros(4, 5).T, torch.zeros(5), ValueError),
])
def test_lift_views_rejects_bad_accumulators(fs, ws, exc):
    from semantic_gaussians_b200.fusion import lift_views
    with pytest.raises(exc):
        lift_views(_Gaussians(), [object()], [torch.zeros(4, 6, 8)], _Pipe, fs, ws)


def test_lift_views_rejects_cpu_tensors():
    from semantic_gaussians_b200.fusion import lift_views
    with pytest.raises(ValueError, match="CUDA"):
        lift_views(_Gaussians(), [object()], [torch.zeros(4, 6, 8)], _Pipe, torch.zeros(5, 4), torch.zeros(5))


def test_lift_scene_needs_semantic_buffers():
    from semantic_gaussians_b200.fusion import lift_scene
    g = _Gaussians()
    g._features_semantic = torch.empty(0)
    with pytest.raises(ValueError, match="create_semantic"):
        lift_scene(g, [object()], [torch.zeros(4, 6, 8)], _Pipe)


def test_lift_scene_passes_map_checks_through():
    from semantic_gaussians_b200.fusion import lift_scene
    g = _Gaussians()
    g._features_semantic, g._times = torch.zeros(5, 4), torch.zeros(5, 1)
    with pytest.raises(TypeError, match="float16 or float32"):
        lift_scene(g, [object()] * 6, [torch.zeros(4, 6, 8, dtype=torch.int8)] * 6, _Pipe)


def _inputs(**kw):
    base = dict(P=10, D=0, M=0, W=64, H=64, C=8, background=None, means3D=1, shs=None, colors_precomp=None,
                opacities=1, scales=1, scale_modifier=1.0, rotations=1, cov3D_precomp=None, viewmatrix=1,
                projmatrix=1, campos=1, tan_fovx=0.5, tan_fovy=0.5, prefiltered=0, debug=0)
    base.update(kw)
    return _lib.ViewInputs(**base)


@pytest.mark.parametrize("kw,V,dtype,maps_null,msg", [
    (dict(), 0, _lib.FEAT_F16, False, b"1 <= V"),
    (dict(), 9, _lib.FEAT_F16, False, b"1 <= V"),
    (dict(C=0), 1, _lib.FEAT_F32, False, b"invalid sizes"),
    (dict(), 1, 7, False, b"dtype"),
    (dict(), 1, _lib.FEAT_F16, True, b"null map"),
    (dict(shs=1, M=1), 1, _lib.FEAT_F16, False, b"must be NULL"),
    (dict(colors_precomp=1), 1, _lib.FEAT_F16, False, b"must be NULL"),
    (dict(background=1), 1, _lib.FEAT_F16, False, b"must be NULL"),
    (dict(cov3D_precomp=1), 1, _lib.FEAT_F32, False, b"scale/rotation"),
    (dict(scales=None), 1, _lib.FEAT_F32, False, b"scale/rotation"),
    (dict(opacities=None), 1, _lib.FEAT_F32, False, b"null required"),
])
def test_lift_batch_validation_happens_before_cuda(kw, V, dtype, maps_null, msg):
    lib = _lib.load()
    cams = (_lib.Camera * 9)(*[_lib.Camera(1, 1, 1, 0.5, 0.5)] * 9)
    maps = (C.c_void_p * 9)(*([None] if maps_null else [1]) * 9)
    # ctx 1 is a dummy: the call must fail before it is dereferenced
    rc = lib.sgb_lift_batch(1, C.byref(_inputs(**kw)), V, cams, maps, dtype, 1, 1, None)
    assert rc == E_INVALID
    assert msg in lib.sgb_last_error(), lib.sgb_last_error()


def test_lift_batch_refuses_null_arrays():
    lib = _lib.load()
    cams = _lib.Camera(1, 1, 1, 0.5, 0.5)
    maps = (C.c_void_p * 1)(1)
    assert lib.sgb_lift_batch(1, C.byref(_inputs()), 1, C.byref(cams), maps, _lib.FEAT_F16, None, 1, None) == E_INVALID
    assert lib.sgb_lift_batch(1, C.byref(_inputs()), 1, C.byref(cams), maps, _lib.FEAT_F16, 1, None, None) == E_INVALID
    assert lib.sgb_lift_batch(1, C.byref(_inputs()), 1, C.byref(cams), None, _lib.FEAT_F16, 1, 1, None) == E_INVALID
    assert lib.sgb_lift_batch(1, C.byref(_inputs()), 1, None, maps, _lib.FEAT_F16, 1, 1, None) == E_INVALID


def test_library_exports_lift_and_the_weight_sum_stage():
    lib = _lib.load()
    assert "sgb_lift_batch" in _lib.EXPORTS and hasattr(lib, "sgb_lift_batch")
    names = [lib.sgb_profile_stage_name(i).decode() for i in range(lib.sgb_profile_num_stages())]
    # appended after the existing stages: their indices do not move
    assert names[12:] == ["alpha_pass", "dfeature", "weight_sum"]


def test_fp16_contraction_loads_its_map_by_tensor_map():
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = {}
    name = None
    for line in sass.splitlines():
        if "Function : " in line:
            name = line.split("Function : ")[1].strip()
            funcs[name] = []
        elif name:
            funcs[name].append(line)
    f16 = [n for n in funcs if "dfeature_persistent_kernel" in n and "__half" in n]
    f32 = [n for n in funcs if "dfeature_persistent_kernel" in n and "IfE" in n]
    assert len(f16) == 1 and len(f32) == 1, list(funcs)
    body = "\n".join(funcs[f16[0]])
    assert "UTMALDG" in body            # the dL (map) tile and the weight slabs arrive by tensor-map copies
    assert "HADD2.F32" in body or "F2F" in body or "HADD2" in body   # widened to fp32 on chip
    assert any("pool_weight_sum_kernel" in n for n in funcs)
