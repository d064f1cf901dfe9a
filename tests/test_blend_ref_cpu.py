"""The float64 blend restatement (tests/blend_ref.py) against the CPU oracle (oracle/raster_oracle.c, pinned to
the compiled reference by test_oracle_cpu.py) on the oracle's own preprocess and binning, and evidence that the
comparison the GPU sweep relies on rejects results that are wrong the way a blend kernel could be wrong."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blend_ref as br  # noqa: E402
from oracle import oracle as orc  # noqa: E402

from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras  # noqa: E402

FRAGILE_MAX = 0.03   # at most this fraction of pixels may be left out (flagged by either side)

# (P, W, H, C, scale_mean, opacity or None, background)
CASES = {
    "c1": (3000, 64, 48, 1, 0.04, None, "ramp"),
    "c3_zero_bg": (3000, 64, 48, 3, 0.04, None, "zero"),
    "c17": (3000, 64, 48, 17, 0.04, None, "ramp"),
    "c64_zero_bg": (3000, 64, 48, 64, 0.04, None, "zero"),
    "ragged_c17": (3000, 61, 37, 17, 0.04, None, "ramp"),
    "dense_faint_c8": (20000, 48, 32, 8, 0.05, 0.02, "ramp"),
}


def _case(name):
    P, W, H, C, scale, opacity, bgkind = CASES[name]
    scene = make_scene(P, seed=31, channels=C, scale_mean=scale)
    if opacity is not None:
        scene.opacity[:] = opacity
    cam = orbit_cameras(4, W, H)[1]
    bg = np.zeros(C, np.float32) if bgkind == "zero" else np.linspace(0.1, 0.6, C).astype(np.float32)
    fo = orc.forward(orc.scene_dict(scene), orc.cam_dict(cam), W, H, bg, features=scene.features)
    pre, b = fo["pre"], fo["bin"]
    st = dict(means2D=torch.from_numpy(pre["means2D"]), conic_opacity=torch.from_numpy(pre["conic_opacity"]),
              point_list=torch.from_numpy(b["point_list"].astype(np.int64)),
              ranges=torch.from_numpy(b["ranges"].astype(np.int64)), features=torch.from_numpy(scene.features),
              bg=torch.from_numpy(bg), W=W, H=H)
    want = br.blend_forward(**st)
    fragile = want["fragile"].numpy() | fo["fragile"].reshape(-1)
    dL = np.random.default_rng(7).standard_normal((C, H * W)).astype(np.float32)
    dL[:, fragile] = 0.0            # a pixel with zero dL/dout adds nothing to any gradient, on either side
    dL = dL.reshape(C, H, W)
    go = orc.backward(fo, orc.scene_dict(scene), orc.cam_dict(cam), W, H, bg, dL, features=scene.features)
    return dict(scene=scene, cam=cam, fo=fo, go=go, st=st, want=want, fragile=fragile, dL=torch.from_numpy(dL))


_cache = {}


def case(name):
    if name not in _cache:
        _cache[name] = _case(name)
    return _cache[name]


def errors(k, fwd, bwd):
    """compare() of the oracle's outputs (got) against an fp64 result (want) over the non-fragile pixels."""
    ok = ~k["fragile"]
    C = fwd["color"].shape[0]
    out = dict(color=br.compare(k["fo"]["color"].reshape(C, -1)[:, ok], fwd["color"].reshape(C, -1)[:, ok]),
               final_T=br.compare(k["fo"]["final_T"][ok], fwd["final_T"][ok]))
    out.update(br.grad_errors(k["go"], bwd))
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_fp64_blend_matches_cpu_oracle(name):
    k = case(name)
    fo, want, ok = k["fo"], k["want"], ~k["fragile"]
    assert k["fragile"].mean() <= FRAGILE_MAX, k["fragile"].mean()
    assert int(fo["n_contrib"].max()) > 0
    assert np.array_equal(fo["n_contrib"][ok].astype(np.int64), want["n_contrib"].numpy()[ok])
    wb = br.blend_backward(**k["st"], dL_dpix=k["dL"])
    errs = errors(k, want, wb)
    assert all(e <= 1.0 for e in errs.values()), errs
    for g in wb.values():
        assert float(g.abs().max()) > 0


def test_dense_faint_scene_has_long_lists():
    k = case("dense_faint_c8")
    rg = k["st"]["ranges"]
    assert int((rg[:, 1] - rg[:, 0]).max()) > 512


def _drop_last_blended_entry(k):
    """The list of one tile without its last blended entry: the tile whose last blended entry still sees the most
    light, so that the entry matters."""
    st, want, W = k["st"], k["want"], k["st"]["W"]
    gx = (W + 15) // 16
    ncon, fT = want["n_contrib"].reshape(-1, W), want["final_T"].reshape(-1, W)
    best = None
    for t, (s, e) in enumerate(st["ranges"].tolist()):
        if e <= s:
            continue
        y0, x0 = (t // gx) * 16, (t % gx) * 16
        n, T = ncon[y0:y0 + 16, x0:x0 + 16], fT[y0:y0 + 16, x0:x0 + 16]
        m = int(n.max())
        if m > 0 and (best is None or float(T[n == m].max()) > best[0]):
            best = (float(T[n == m].max()), t, s + m - 1)
    _, t, drop = best
    pl = torch.cat([st["point_list"][:drop], st["point_list"][drop + 1:]])
    rg = st["ranges"].clone()
    rg[t, 1] -= 1
    rg[rg[:, 0] > drop] -= 1          # the later tiles (empty tiles keep (0, 0))
    return dict(st, point_list=pl, ranges=rg)


def _wrong(k, kind):
    st, dL = k["st"], k["dL"]
    fwd = k["want"]
    if kind == "tile_list_entry_dropped":
        st2 = _drop_last_blended_entry(k)
        return br.blend_forward(**st2), br.blend_backward(**st2, dL_dpix=dL)
    if kind == "transmittance_one_entry_early":
        return fwd, br.blend_backward(**st, dL_dpix=dL, _t_one_entry_early=True)
    if kind == "background_term_left_out":
        return fwd, br.blend_backward(**dict(st, bg=torch.zeros_like(st["bg"])), dL_dpix=dL)
    bwd = br.blend_backward(**st, dL_dpix=dL)
    if kind == "conic_y_without_half":
        bwd["dL_dconic"][:, 1] *= 2.0
    elif kind == "two_channels_swapped":
        g = bwd["dL_dcolors"]
        r = int(g.abs().amax(dim=1).argmax())
        i, j = int(g[r].argmax()), int(g[r].argmin())
        g[r, [i, j]] = g[r, [j, i]]
    return fwd, bwd


@pytest.mark.parametrize("kind", ["tile_list_entry_dropped", "transmittance_one_entry_early",
                                  "background_term_left_out", "conic_y_without_half", "two_channels_swapped"])
def test_comparison_rejects_wrong_results(kind):
    k = case("c17")
    assert float(k["st"]["bg"].abs().max()) > 0
    fwd, bwd = _wrong(k, kind)
    errs = errors(k, fwd, bwd)
    assert max(errs.values()) > 1.0, errs
