"""The blend stage of the reference rasterizer restated in float64 for the tests: the front-to-back walk of
channel-rasterization/cuda_rasterizer/forward.cu:283-371 and the gradients of backward.cu:394-552, evaluated on a
kernel's own per-Gaussian state (means2D, conic_opacity) and tile lists (point_list, ranges).  Nothing here decides
anything differently from the fp32 program except where fp32 rounding could: those pixels are reported as fragile,
so that a test can leave them out and measure nothing but the kernel's own arithmetic error.

The walk is vectorised per 16 x 16 tile: (pixels x list entries) matrices for alpha and the transmittance, one
reverse cumulative sum for the back-to-front term, and dot products s = <feature, dL/dpixel> so that no
(pixels x entries x channels) array is built.  Every function runs on CPU and CUDA tensors alike."""
from __future__ import annotations

import numpy as np
import torch

TILE = 16
# the fp32 constants of the walk, exactly (forward.cu:344,345,348)
ALPHA_MAX = float(np.float32(0.99))
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))
T_MIN = float(np.float32(0.0001))

# Fragile bands.  The fp32 power -0.5 (a dx^2 + c dy^2) - b dx dy carries an absolute error of a few ulp of
# mag = 0.5 (|a| dx^2 + |c| dy^2) + |b dx dy| (the rounding of dx included); G = exp(power) inherits it as a
# relative error, plus the error of expf / __expf (under 1e-6 relative for |power| <= 30).  Both bands below are
# more than ten times those bounds.  The transmittance is a product of up to thousands of factors (1 - alpha),
# each of which carries alpha / (1 - alpha) times the relative error of its alpha: its band is that sum, taken
# along the list.
EPS32 = 2.0 ** -24
POWER_ULPS = 64.0
G_REL = 1e-5
T_ULPS = 8.0

# Kernel against this restatement: every entry must satisfy |got - want| <= RTOL |want| + ATOL_SCALE max|want|.
# Set once from the configurations that are also pinned to the compiled reference (the largest error measured
# there on an H100 80GB HBM3 at 700 W is 0.25 of it, in dL_dconic); applies to every case.
RTOL = 1e-4
ATOL_SCALE = 1e-5


def compare(got, want, rtol=RTOL, atol_scale=ATOL_SCALE) -> float:
    """max over entries of |got - want| / (rtol |want| + atol_scale max|want|): the arrays agree when this is
    <= 1, i.e. when every entry is within tolerance.  There is no allowance for a fraction of bad entries."""
    got = torch.as_tensor(got).detach().to(dtype=torch.float64, device="cpu").reshape(-1)
    want = torch.as_tensor(want).detach().to(dtype=torch.float64, device="cpu").reshape(-1)
    assert got.shape == want.shape, (got.shape, want.shape)
    if want.numel() == 0:
        return 0.0
    diff = (got - want).abs()
    if not bool(torch.isfinite(diff).all()):
        return float("inf")
    tol = rtol * want.abs() + atol_scale * want.abs().max()
    return float(torch.where(diff == 0, torch.zeros_like(diff), diff / tol).max())   # diff > 0 = tol: inf


def _tiles(ranges, W, H, tile_rows):
    """(tile id, list start, list end, pixel x, pixel y) of every non-empty tile in tile rows [r0, r1)."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    r0, r1 = tile_rows if tile_rows is not None else (0, gy)
    rg = ranges.reshape(-1, 2)[r0 * gx:min(r1, gy) * gx].to("cpu", torch.int64).tolist()
    for k, (s, e) in enumerate(rg):
        if e <= s:
            continue
        t = r0 * gx + k
        x0, y0 = (t % gx) * TILE, (t // gx) * TILE
        ys, xs = torch.meshgrid(torch.arange(y0, min(y0 + TILE, H)), torch.arange(x0, min(x0 + TILE, W)),
                                indexing="ij")
        yield t, s, e, xs.reshape(-1), ys.reshape(-1)


def _walk(mean, con, ids, px, py):
    """forward.cu:328-366 for the pixels (px, py) of one tile over its list entries ids, in float64."""
    dev = mean.device
    px, py = px.to(dev, torch.float64), py.to(dev, torch.float64)
    dx = mean[ids, 0][None, :] - px[:, None]               # d = xy - pixf, no half-pixel offset (forward.cu:334)
    dy = mean[ids, 1][None, :] - py[:, None]
    ca, cb, cc, op = (con[ids, k][None, :] for k in range(4))
    qa, qc, qb = ca * dx * dx, cc * dy * dy, cb * dx * dy
    power = -0.5 * (qa + qc) - qb
    mag = 0.5 * (qa.abs() + qc.abs()) + qb.abs()
    G = torch.exp(power)
    oG = op * G
    alpha = oG.clamp(max=ALPHA_MAX)
    valid = (power <= 0) & (alpha >= ALPHA_MIN)             # :336-346 (power > 0 and alpha < 1/255 skip)
    a = torch.where(valid, alpha, torch.zeros_like(alpha))
    incl = torch.cumprod(1.0 - a, dim=1)                    # T after each entry
    excl = torch.cat([torch.ones_like(incl[:, :1]), incl[:, :-1]], dim=1)   # T in front of each entry
    n, L = a.shape
    pos = torch.arange(L, device=dev)
    # the first entry whose test_T falls below 1e-4 ends the walk (:347-351); at a skipped entry T is unchanged,
    # so that first entry is always a blended one
    stopped = incl < T_MIN
    has_stop = stopped.any(dim=1)
    stop = torch.where(has_stop, stopped.to(torch.int8).argmax(dim=1), torch.full_like(has_stop, L, dtype=torch.int64))
    contrib = valid & (pos[None, :] < stop[:, None])
    w = torch.where(contrib, a * excl, torch.zeros_like(a))
    final_T = torch.where(has_stop, excl.gather(1, stop.clamp(max=L - 1)[:, None])[:, 0], incl[:, -1])
    n_contrib = torch.where(contrib, pos[None, :] + 1, torch.zeros_like(pos)[None, :]).amax(dim=1)

    # fragile: a decision of an entry the walk reaches sits within fp32 rounding of its threshold
    seen = pos[None, :] <= stop[:, None]
    e_pow = POWER_ULPS * EPS32 * mag
    e_g = G_REL + e_pow
    e_T = torch.cumsum(torch.where(valid, a / (1.0 - a) * e_g + T_ULPS * EPS32, torch.zeros_like(a)), dim=1)
    near = ((power.abs() <= e_pow) & (mag > 0)
            | ((oG - ALPHA_MIN).abs() <= e_g * oG)
            | ((oG - ALPHA_MAX).abs() <= e_g * oG)
            | (valid & ((incl - T_MIN).abs() <= e_T * incl)))
    fragile = (near & seen).any(dim=1)
    return dict(dx=dx, dy=dy, ca=ca, cb=cb, cc=cc, op=op, G=G, a=a, excl=excl, w=w, contrib=contrib,
                final_T=final_T, n_contrib=n_contrib, fragile=fragile)


def _f64(t, dev):
    return torch.as_tensor(t).to(device=dev, dtype=torch.float64)


def blend_forward(means2D, conic_opacity, point_list, ranges, features, bg, W, H, tile_rows=None):
    """The blend of one view.  means2D (P, 2), conic_opacity (P, 4), features (P, C), bg (C) as the fp32 arrays
    the kernel reads; point_list (R,), ranges (tiles, 2).  Returns float64 color (C, H, W), final_T (H W),
    n_contrib (H W) int64 and fragile (H W) bool.  With tile_rows = (r0, r1) only those tile rows are evaluated
    and every other pixel is left zero."""
    dev = torch.as_tensor(means2D).device
    mean, con = _f64(means2D, dev).reshape(-1, 2), _f64(conic_opacity, dev).reshape(-1, 4)
    feat, bgc = _f64(features, dev), _f64(bg, dev).reshape(-1)
    pl = torch.as_tensor(point_list).to(dev, torch.int64).reshape(-1)
    C = feat.shape[1]
    color = torch.zeros((C, H * W), dtype=torch.float64, device=dev)
    final_T = torch.zeros(H * W, dtype=torch.float64, device=dev)
    n_contrib = torch.zeros(H * W, dtype=torch.int64, device=dev)
    fragile = torch.zeros(H * W, dtype=torch.bool, device=dev)
    # a pixel of an empty tile is the background (T = 1)
    gy = (H + TILE - 1) // TILE
    r0, r1 = tile_rows if tile_rows is not None else (0, gy)
    rows = slice(r0 * TILE * W, min(r1 * TILE, H) * W)
    color[:, rows] = bgc[:, None]
    final_T[rows] = 1.0
    for _, s, e, px, py in _tiles(ranges, W, H, tile_rows):
        ids = pl[s:e]
        k = _walk(mean, con, ids, px, py)
        pix = (py * W + px).to(dev)
        color[:, pix] = (k["w"] @ feat[ids] + k["final_T"][:, None] * bgc[None, :]).T   # forward.cu:370-373
        final_T[pix], n_contrib[pix], fragile[pix] = k["final_T"], k["n_contrib"], k["fragile"]
    return dict(color=color.reshape(C, H, W), final_T=final_T, n_contrib=n_contrib, fragile=fragile)


def blend_backward(means2D, conic_opacity, point_list, ranges, features, bg, W, H, dL_dpix, tile_rows=None,
                   _t_one_entry_early=False):
    """backward.cu:394-552 for the blend above and dL/dout dL_dpix (C, H, W), as the reference writes it (in
    particular dL/dG = o dL/dalpha also where alpha is clamped at 0.99).  float64 gradients in the layout of
    sgb_view_grads: dL_dmeans2D (P, 3) with the 0.5 W / 0.5 H factors (:455-456, z stays 0), dL_dconic (P, 4) as
    (x, y, _, w) with y = sum -0.5 gdx dy dL/dG (:544-546), dL_dopacity (P,) and dL_dcolors (P, C).
    _t_one_entry_early uses the transmittance behind each entry instead of the one in front of it: a wrong
    result for the tests that show the comparison would catch such a bug."""
    dev = torch.as_tensor(means2D).device
    mean, con = _f64(means2D, dev).reshape(-1, 2), _f64(conic_opacity, dev).reshape(-1, 4)
    feat, bgc = _f64(features, dev), _f64(bg, dev).reshape(-1)
    pl = torch.as_tensor(point_list).to(dev, torch.int64).reshape(-1)
    P, C = feat.shape
    dL = _f64(dL_dpix, dev).reshape(C, H * W)
    g_mean = torch.zeros((P, 3), dtype=torch.float64, device=dev)
    g_conic = torch.zeros((P, 4), dtype=torch.float64, device=dev)
    g_opac = torch.zeros(P, dtype=torch.float64, device=dev)
    g_feat = torch.zeros((P, C), dtype=torch.float64, device=dev)
    for _, s, e, px, py in _tiles(ranges, W, H, tile_rows):
        ids = pl[s:e]
        k = _walk(mean, con, ids, px, py)
        pix = (py * W + px).to(dev)
        dLp = dL[:, pix].T                                   # (pixels, C)
        w, a, T = k["w"], k["a"], k["excl"]
        if _t_one_entry_early:
            T = T * (1.0 - a)
            w = torch.where(k["contrib"], a * T, torch.zeros_like(w))
        g_feat.index_add_(0, ids, w.T @ dLp)                 # dchannel_dcolor = alpha T (:499, :519)
        # accum_rec of entry i is sum_{j > i} w_j c_j / (T_i (1 - alpha_i)), so
        # dL/dalpha_i = T_i <c_i, dL> - (sum_{j > i} w_j <c_j, dL> + T_final <bg, dL>) / (1 - alpha_i)  (:505-530)
        sdot = dLp @ feat[ids].T                             # (pixels, entries)
        ws = w * sdot
        behind = torch.flip(torch.cumsum(torch.flip(ws, [1]), 1), [1]) - ws
        bgdot = dLp @ bgc
        dL_dalpha = T * sdot - (behind + k["final_T"][:, None] * bgdot[:, None]) / (1.0 - a)
        dL_dalpha = torch.where(k["contrib"], dL_dalpha, torch.zeros_like(dL_dalpha))
        dL_dG = k["op"] * dL_dalpha                          # :533
        gdx, gdy = k["G"] * k["dx"], k["G"] * k["dy"]
        dG_ddelx = -gdx * k["ca"] - gdy * k["cb"]
        dG_ddely = -gdy * k["cc"] - gdx * k["cb"]
        g_mean[:, 0].index_add_(0, ids, (dL_dG * dG_ddelx).sum(0) * (0.5 * W))
        g_mean[:, 1].index_add_(0, ids, (dL_dG * dG_ddely).sum(0) * (0.5 * H))
        g_conic[:, 0].index_add_(0, ids, (-0.5 * gdx * k["dx"] * dL_dG).sum(0))
        g_conic[:, 1].index_add_(0, ids, (-0.5 * gdx * k["dy"] * dL_dG).sum(0))
        g_conic[:, 3].index_add_(0, ids, (-0.5 * gdy * k["dy"] * dL_dG).sum(0))
        g_opac.index_add_(0, ids, (k["G"] * dL_dalpha).sum(0))
    return dict(dL_dmeans2D=g_mean, dL_dconic=g_conic, dL_dopacity=g_opac, dL_dcolors=g_feat)


# what of each sgb_view_grads array the blend writes
GRAD_COLUMNS = dict(dL_dmeans2D=[0, 1], dL_dconic=[0, 1, 3], dL_dopacity=None, dL_dcolors=None)


def grad_errors(got: dict, want: dict, rtol=RTOL, atol_scale=ATOL_SCALE) -> dict:
    """compare() of the four blend gradients (got may hold (P, 2, 2) conic buffers or (P, 1) opacities)."""
    out = {}
    for name, cols in GRAD_COLUMNS.items():
        g = torch.as_tensor(got[name]).reshape(want[name].shape[0], -1)
        wv = want[name].reshape(want[name].shape[0], -1)
        if cols is not None:
            g, wv = g[:, cols], wv[:, cols]
        out[name] = compare(g, wv, rtol, atol_scale)
    return out
