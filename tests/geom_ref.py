"""The per-Gaussian geometry stage of the reference rasterizer restated in float64 for the tests: the forward of
channel-rasterization/cuda_rasterizer/forward.cu:20-256 with auxiliary.h:41-164 (near cull, 3-D and 2-D covariance,
conic, radius, tile rectangle, SH colour) and the backward of backward.cu:20-136 (SH colour), :141-271 (screen
covariance and the covariance path of dL/dmean), :275-336 (scale and rotation) and :341-391 (projected centre).
It restates the reference's own expanded expressions, not the product's matrix-calculus form
(semantic-gaussians_b200/csrc/geom_grad.cuh), so that the two derivations stay independent.

Every float output comes with a magnitude companion: values are carried as `AV` (value, magnitude) pairs, and
the magnitude is the first-order running bound of fp32 rounding, in units of 2^-24:
    m(x) = |x| for an input,  m(a +- b) = m_a + m_b,  m(a b) = m_a |b| + |a| m_b,
    m(a / b) = (m_a + |a / b| m_b) / |b|,  m(sqrt a) = sqrt(a) + m_a / (2 sqrt a).
For a sum of products of inputs this is twice the sum of the absolute values of its terms; an fp32 program that
evaluates the same quantity, in any order of its terms and with or without FMA contraction, differs from it by a
small multiple of 2^-24 m.  A quotient by a cancelling denominator carries the denominator's magnitude, so every
output behind the conic inversion is scaled by the 2-D conditioning kappa = (|a c| + b^2) / |a c - b^2| of the
screen covariance through m(det) / |det|; `geom_forward` also reports kappa.  A kernel entry passes when
|got - want| <= RTOL * magnitude.  This is the per-entry bound RTOL * kappa * sum|terms| generalised: the running
bound follows each intermediate through the whole chain, so terms that cancel and quotients by a cancelling
denominator anywhere along it (not only at the conic inversion) widen the tolerance of exactly the entries they
reach.

Integer outputs (the cull, radius, tile rectangle, tiles_touched, clamped flags) are decided exactly here.  Where a
decision's argument lies within fp32 rounding of its threshold the Gaussian is reported as fragile, so that a test
can leave it out and measure nothing but the kernel's arithmetic.  Every function runs on CPU and CUDA tensors."""
from __future__ import annotations

import numpy as np
import torch

TILE = 16
EPS32 = 2.0 ** -24


def _c(x) -> float:
    """An fp32 constant of the reference's code, exactly."""
    return float(np.float32(x))


NEAR_Z = _c(0.2)          # auxiliary.h:154
W_EPS = _c(0.0000001)     # auxiliary.h:150, backward.cu:369
LOWPASS = _c(0.3)         # forward.cu:110-111, backward.cu:194-196
DET_REG = _c(0.0000001)   # backward.cu:200
EIG_FLOOR = _c(0.1)       # forward.cu:230-231
SH_C0 = _c(0.28209479177387814)
SH_C1 = _c(0.4886025119029199)
SH_C2 = [_c(v) for v in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                         0.5462742152960396)]
SH_C3 = [_c(v) for v in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                         -0.4570457994644658, 1.445305721320277, -0.5900435899266435)]

# Fragile band: a decision whose argument q lies within BAND_ULPS * 2^-24 * magnitude(q) of its threshold.  The
# fp32 oracle and the kernels stay within 2^-24 * 1.6 magnitude of every output (below), so the band is ten times
# the largest rounding error measured; its magnitude grows where the argument is ill-conditioned (the radius of a
# large, nearly isotropic Gaussian, whose eigenvalue comes from the square root of a cancelling difference).
BAND_ULPS = 16.0

# Kernel (or fp32 oracle) against this restatement: every entry must satisfy |got - want| <= RTOL * magnitude.
# Set once from the scenes and cameras on which the kernels are pinned to the compiled reference
# (test_geom_fp64_gpu.py's SH calibration cases, test_blend_fp64_gpu.py's feature ones; their dL/dout is drawn by
# the tests), measured on an H100 80GB HBM3 at a 700 W power limit:
# their largest error is 0.075 RTOL (depth; 0.059 for dL_dmeans3D, the largest gradient), i.e. 1.2 * 2^-24 times
# the magnitude, and 0.10 RTOL across every other GPU case.  The fp32 CPU oracle stays within 0.08 RTOL and the
# host build of geom_grad.cuh within 0.06 RTOL: RTOL is ten times the largest error measured.
RTOL = 16 * EPS32


class AV:
    """A float64 value and its magnitude companion (see the module docstring)."""
    __slots__ = ("v", "m")

    def __init__(self, v, m=None):
        self.v = v
        self.m = v.abs() if m is None else m

    @staticmethod
    def _lift(o):
        if isinstance(o, AV):
            return o
        return AV(o, abs(o) if isinstance(o, float) else o.abs())

    def __add__(self, o):
        o = AV._lift(o)
        return AV(self.v + o.v, self.m + o.m)

    __radd__ = __add__

    def __sub__(self, o):
        o = AV._lift(o)
        return AV(self.v - o.v, self.m + o.m)

    def __rsub__(self, o):
        return AV._lift(o) - self

    def __neg__(self):
        return AV(-self.v, self.m)

    def __mul__(self, o):
        o = AV._lift(o)
        return AV(self.v * o.v, self.m * abs(o.v) + abs(self.v) * o.m)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = AV._lift(o)
        if isinstance(o.v, float):
            return AV(self.v / o.v, self.m / abs(o.v))
        q = self.v / o.v
        return AV(q, (self.m + q.abs() * o.m) / o.v.abs())

    def __rtruediv__(self, o):
        return AV._lift(o) / self

    def sqrt(self):
        r = self.v.sqrt()
        return AV(r, r + 0.5 * self.m / r)

    def __getitem__(self, k):
        return AV(self.v[k], self.m[k])


def stack(avs, dim=-1) -> AV:
    return AV(torch.stack([a.v for a in avs], dim), torch.stack([a.m for a in avs], dim))


def _where(cond, a: AV, b: AV) -> AV:
    return AV(torch.where(cond, a.v, b.v), torch.where(cond, a.m, b.m))


def _f64(t, dev):
    return torch.as_tensor(t).to(device=dev, dtype=torch.float64)


def _exact(t, dev) -> AV:
    v = _f64(t, dev)
    return AV(v, v.abs())


def _near(q: AV, k, extra=0.0):
    """q lies within the fragile band of the threshold k."""
    return (q.v - k).abs() <= BAND_ULPS * EPS32 * q.m + extra


def _camera(view, proj, campos, W, H, tan_fovx, tan_fovy):
    vm = [float(x) for x in np.asarray(view, np.float32).reshape(-1)]
    pm = [float(x) for x in np.asarray(proj, np.float32).reshape(-1)]
    cp = [float(x) for x in np.asarray(campos, np.float32).reshape(-1)]
    tx, ty = np.float32(tan_fovx), np.float32(tan_fovy)
    # rasterizer_impl.cu:223-224 and forward.cu:82-83, fp32 as the kernels compute them
    return dict(view=vm, proj=pm, campos=cp, fx=float(np.float32(W) / (np.float32(2.0) * tx)),
                fy=float(np.float32(H) / (np.float32(2.0) * ty)), limx=float(np.float32(1.3) * tx),
                limy=float(np.float32(1.3) * ty))


def _view_point(m, p):
    """transformPoint4x3 (auxiliary.h:58-66): m column-major, element (row i, col j) at m[4 j + i]."""
    return [m[i] * p[0] + m[4 + i] * p[1] + m[8 + i] * p[2] + m[12 + i] for i in range(3)]


def _hom(m, p):
    """transformPoint4x4 (auxiliary.h:68-77)."""
    return [m[i] * p[0] + m[4 + i] * p[1] + m[8 + i] * p[2] + m[12 + i] for i in range(4)]


def _clamp_t(t, cam):
    """forward.cu:80-87 / backward.cu:163-173: the Jacobian's evaluation point clamped to 1.3 tan(fov / 2) sideways.
    Returns the clamped (tx, ty), the pass masks and the two ratios."""
    out, passes, ratios = [], [], []
    for k, lim in ((0, cam["limx"]), (1, cam["limy"])):
        r = t[k] / t[2]
        inside = (r.v >= -lim) & (r.v <= lim)
        rc = _where(inside, r, AV(r.v.clamp(-lim, lim), torch.full_like(r.m, lim)))
        out.append(rc * t[2])
        passes.append(inside)
        ratios.append(r)
    return out, passes, ratios


def _T(t, tcl, cam):
    """The upper 2 x 3 of T = W J (forward.cu:89-99): T[i][j] in glm's [column][row], i.e. row i of J W^T."""
    v, fx, fy = cam["view"], cam["fx"], cam["fy"]
    tz2 = t[2] * t[2]
    J00, J02 = fx / t[2], -(fx * tcl[0]) / tz2
    J11, J12 = fy / t[2], -(fy * tcl[1]) / tz2
    return [[v[4 * r] * J00 + v[4 * r + 2] * J02 for r in range(3)],
            [v[4 * r + 1] * J11 + v[4 * r + 2] * J12 for r in range(3)]]


def _sym(cov6):
    c = cov6
    return [[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]]


def _rotation(q, quat_order=(0, 1, 2, 3)):
    """forward.cu:127-137: R as glm::mat3 (R[column][row]) from q = (r, x, y, z), used as given (not normalised)."""
    r, x, y, z = (q[i] for i in quat_order)
    return [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - r * z), 2.0 * (x * z + r * y)],
            [2.0 * (x * y + r * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - r * x)],
            [2.0 * (x * z - r * y), 2.0 * (y * z + r * x), 1.0 - 2.0 * (x * x + y * y)]], (r, x, y, z)


def _cov3d(scales, rotations, mod, dev):
    """forward.cu:118-151: Sigma = M^T M with M = S R, S = diag(mod * scale)."""
    s = [_exact(scales[:, k], dev) * mod for k in range(3)]
    R, _ = _rotation([_exact(rotations[:, k], dev) for k in range(4)])
    M = [[s[r] * R[c][r] for r in range(3)] for c in range(3)]         # (S R)[c][r] = s_r R[c][r]
    Sig = lambda c, r: M[r][0] * M[c][0] + M[r][1] * M[c][1] + M[r][2] * M[c][2]   # (M^T M)[c][r]
    return [Sig(0, 0), Sig(0, 1), Sig(0, 2), Sig(1, 1), Sig(1, 2), Sig(2, 2)]


def _sh_dir(means, campos, dev):
    p = [_exact(means[:, k], dev) for k in range(3)]
    d = [p[k] - campos[k] for k in range(3)]
    ln = (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]).sqrt()
    return d, [d[k] / ln for k in range(3)]


def _sh_basis(D, x, y, z):
    """forward.cu:30-60: the basis functions Y_k in the reference's order and signs, k < (D + 1)^2."""
    Y = [AV(torch.full_like(x.v, SH_C0))]
    if D > 0:
        Y += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if D > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        Y += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2.0 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
    if D > 2:
        Y += [SH_C3[0] * y * (3.0 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4.0 * zz - xx - yy),
              SH_C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy), SH_C3[4] * x * (4.0 * zz - xx - yy),
              SH_C3[5] * z * (xx - yy), SH_C3[6] * x * (xx - 3.0 * yy)]
    return Y


def _col(a: AV) -> AV:
    return AV(a.v[:, None], a.m[:, None])


def _rect_edge(e: AV, gmax, dev):
    """getRect (auxiliary.h:46-56) of one edge: min(grid, max(0, (int) e)), truncation toward zero; fragile where e
    lies within the band of an integer k that the clamp does not hide (1 <= k <= grid)."""
    val = torch.trunc(e.v).clamp(0, gmax).to(torch.int64)
    k = torch.round(e.v)
    return val, _near(e, k) & (k >= 1) & (k <= gmax)


AA_DILATION = LOWPASS        # the 0.3 px^2 the anti-aliasing filter compensates for
AA_FLOOR = _c(2.5e-5)       # the floor of det C0 / det C


def _aa_factor(a0, b, c0):
    """3DGS's anti-aliasing opacity factor (forward.cu of the 3DGS rasterizer with antialiasing) in scalar form:
        det C0 = a0 c0 - b^2,  det C = (a0 + 0.3) (c0 + 0.3) - b^2,  h = sqrt(max(2.5e-5, det C0 / det C)).
    Returns (h as AV, active = r above the floor, fragile band of that decision).  det C0 cancels for needles and
    sub-pixel Gaussians, and its magnitude (|a0 c0| + b^2) carries that into r, h and everything formed from them.
    On the floor branch h is the constant sqrt(2.5e-5), whose fp32 rounding its own magnitude covers."""
    det0 = a0 * c0 - b * b
    detc = (a0 + AA_DILATION) * (c0 + AA_DILATION) - b * b
    r = det0 / detc
    active = r.v > AA_FLOOR
    floor = AV(torch.full_like(r.v, AA_FLOOR ** 0.5))
    h = _where(active, AV(r.v.clamp(min=AA_FLOOR), r.m).sqrt(), floor)
    return h, active, _near(r, AA_FLOOR)


def _aa_dr(a0, b, c0, mutation=None):
    """dr/d(a0, b, c0) of r = det C0 / det C, b the off-diagonal value (one variable that appears twice in C): 3DGS's
    backward.cu expression with x = a0, y = c0, z = b, w = 0.3:
        dr/dx = w (w y + y^2 + z^2) / den^2,  dr/dy = w (w x + x^2 + z^2) / den^2,  dr/dz = -2 w z (w + x + y) / den^2,
    den = w^2 + w (x + y) + x y - z^2 = det C."""
    w, x, y, z = AA_DILATION, a0, c0, b
    den = w * w + w * (x + y) + x * y - z * z
    if mutation == "aa_det_swapped":    # det C0 where det C belongs
        den = x * y - z * z
    den2 = den * den
    dz = -2.0 * w * z * (w + x + y) / den2
    if mutation == "aa_offdiag_not_halved":   # the symmetric-matrix entry given the whole dr/db
        dz = 2.0 * dz
    return w * (w * y + y * y + z * z) / den2, dz, w * (w * x + x * x + z * z) / den2


def geom_forward(means3D, opacities, view, proj, campos, W, H, tan_fovx, tan_fovy, *, scales=None, rotations=None,
                 scale_modifier=1.0, cov3D_precomp=None, shs=None, D=0, antialiasing=False):
    """forward.cu:155-256 for every Gaussian.  Inputs are the fp32 arrays the kernel read.  Returns AV outputs
    depth (P,), means2D (P, 2), conic (P, 3), cov3D (P, 6) (from scale / rotation only), rgb (P, 3) (SH only),
    the integers radii, tiles_touched, rect (P, 4) = (xmin, ymin, xmax, ymax), clamped (P, 3), the masks near
    (culled by the near plane) and visible (radius > 0), kappa, and fragile (P,).  With antialiasing also AV aa_h
    (the opacity factor h, unsigned), aa_opacity (o h) and aa_cov0 (P, 3) = (a0, b, c0), the mask aa_active (r above
    the floor), and r within the fragile band of the floor makes a Gaussian fragile (see _aa_factor)."""
    dev = torch.as_tensor(means3D).device
    cam = _camera(view, proj, campos, W, H, tan_fovx, tan_fovy)
    P = means3D.shape[0]
    p = [_exact(means3D[:, k], dev) for k in range(3)]
    t = _view_point(cam["view"], p)
    near = t[2].v <= NEAR_Z
    fragile = _near(t[2], NEAR_Z)
    hom = _hom(cam["proj"], p)
    p_w = 1.0 / (hom[3] + W_EPS)
    ndc = [hom[0] * p_w, hom[1] * p_w]
    if cov3D_precomp is not None:
        cov6 = [_exact(cov3D_precomp[:, k], dev) for k in range(6)]
    else:
        cov6 = _cov3d(scales, rotations, _c(scale_modifier), dev)
    # computeCov2D (forward.cu:74-113): cov = T^T Vrk^T T + 0.3 I, of which (a, b, c) = ([0][0], [0][1], [1][1])
    tcl, passes, ratios = _clamp_t(t, cam)
    for r, lim in zip(ratios, (cam["limx"], cam["limy"])):
        fragile |= _near(AV(r.v.abs(), r.m), lim)
    T = _T(t, tcl, cam)
    V = _sym(cov6)
    TV = [[T[i][0] * V[0][j] + T[i][1] * V[1][j] + T[i][2] * V[2][j] for j in range(3)] for i in range(2)]
    a0 = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2]
    b = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2]
    c0 = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2]
    a, c = a0 + LOWPASS, c0 + LOWPASS
    det = a * c - b * b                                                  # forward.cu:219-223
    det_inv = 1.0 / det
    conic = [c * det_inv, -b * det_inv, a * det_inv]
    kappa = ((a.v * c.v).abs() + b.v * b.v) / (a.v * c.v - b.v * b.v).abs()
    mid = 0.5 * (a + c)                                                  # forward.cu:229-232
    disc = mid * mid - det
    # max(0.1, disc): the floor is exact, but whether it applies is as uncertain as disc itself
    disc = AV(disc.v.clamp(min=EIG_FLOOR), disc.m)
    lam1 = mid + disc.sqrt()
    ext = 3.0 * lam1.sqrt()                                              # lambda1 >= lambda2 always
    fragile |= _near(ext, torch.round(ext.v))
    radius = torch.ceil(ext.v)
    # ndc2Pix (auxiliary.h:41-44) and getRect with the integer radius
    pix = [((ndc[0] + 1.0) * float(W) - 1.0) * 0.5, ((ndc[1] + 1.0) * float(H) - 1.0) * 0.5]
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    rect, edge_frag = [], []
    for e, g in (((pix[0] - radius) / float(TILE), gx), ((pix[1] - radius) / float(TILE), gy),
                 ((pix[0] + radius + float(TILE - 1)) / float(TILE), gx),
                 ((pix[1] + radius + float(TILE - 1)) / float(TILE), gy)):
        val, fr = _rect_edge(e, g, dev)
        rect.append(val)
        edge_frag.append(fr)
    rect = torch.stack(rect, 1)
    tiles = (rect[:, 3] - rect[:, 1]) * (rect[:, 2] - rect[:, 0])
    visible = ~near & (tiles > 0)
    for fr in edge_frag:
        fragile |= fr & ~near
    out = dict(depth=t[2], means2D=stack(pix), conic=stack(conic), kappa=kappa, near=near, visible=visible,
               radii=torch.where(visible, radius, torch.zeros_like(radius)).to(torch.int64),
               tiles_touched=torch.where(visible, tiles, torch.zeros_like(tiles)), rect=rect,
               opacity=_f64(opacities, dev).reshape(-1))
    if cov3D_precomp is None:
        out["cov3D"] = stack(cov6)
    if antialiasing:
        h, active, band = _aa_factor(a0, b, c0)
        fragile |= band & visible
        out.update(aa_h=h, aa_active=active, aa_cov0=stack([a0, b, c0]),
                   aa_opacity=_exact(out["opacity"], dev) * h)
    if shs is not None:
        # computeColorFromSH (forward.cu:20-71)
        _, d = _sh_dir(means3D, cam["campos"], dev)
        Y = _sh_basis(D, *d)
        sh = _f64(shs, dev)
        res = AV(torch.zeros((P, 3), dtype=torch.float64, device=dev))
        for k, y in enumerate(Y):
            res = res + _col(y) * _exact(sh[:, k], dev)
        res = res + 0.5
        out["clamped"] = res.v < 0
        out["rgb"] = AV(res.v.clamp(min=0.0), res.m)
        fragile |= (_near(res, 0.0) & visible[:, None]).any(1)
    out["fragile"] = fragile & ~(near & ~_near(t[2], NEAR_Z))
    return out


# mutations of the backward, each a plausible kernel bug (tests/test_geom_ref_cpu.py and
# tests/test_antialias_ref_cpu.py show the comparison rejects them)
AA_MUTATIONS = ("aa_offdiag_not_halved", "aa_cov_on_floor", "aa_dopacity_not_scaled", "aa_det_swapped",
                "aa_h_squared")
MUTATIONS = ("no_clamp_mask", "conic_xy_not_halved", "cov_offdiag_not_doubled", "scale_times_modifier",
             "quat_xyzw", "no_sh_direction", "clamped_not_zeroed", "y1_sign")


def geom_backward(means3D, radii, view, proj, campos, W, H, tan_fovx, tan_fovy, cov3D, dL_dmeans2D, dL_dconic, *,
                  scales=None, rotations=None, scale_modifier=1.0, shs=None, D=0, clamped=None, dL_dcolors=None,
                  det_reg=True, mutation=None, antialiasing=False, opacities=None, dL_dopacity=None):
    """backward.cu:20-391 for every Gaussian with radii > 0, on the inputs the geometry kernel reads: the fp32 cov3D
    of the forward state (or cov3D_precomp), clamped flags, and the blend's dL_dmeans2D (P, 3) (NDC units),
    dL_dconic (P, 4) (x, y, _, w, with y halved as the blend writes it) and dL_dcolors (P, 3).  Returns AV
    dL_dmeans3D (P, 3), dL_dcov3D (P, 6), and with scale / rotation dL_dscales (P, 3), dL_drotations (P, 4), with
    SH dL_dsh (P, M, 3); Gaussians with radii == 0 get exact zeros.  det_reg=False drops the 1e-7 of
    backward.cu:200 (for finite differences of geom_forward).  mutation: one of MUTATIONS or AA_MUTATIONS.
    antialiasing: dL_dopacity (P,) is g = dL/d(o h), the blend's gradient of the opacity it read, and opacities (P,)
    the raw o.  Returns also AV dL_dopacity = h g, and on the branch above the floor (o g / (2 h)) dr/d(a0, b, c0)
    joins dL/d(a, b, c) before the covariance -> means3D / cov3D / scale / rotation chain (nothing on the floor)."""
    assert mutation is None or mutation in MUTATIONS + AA_MUTATIONS, mutation
    assert not antialiasing or (opacities is not None and dL_dopacity is not None)
    dev = torch.as_tensor(means3D).device
    cam = _camera(view, proj, campos, W, H, tan_fovx, tan_fovy)
    vm, pm, fx, fy = cam["view"], cam["proj"], cam["fx"], cam["fy"]
    P = means3D.shape[0]
    p = [_exact(means3D[:, k], dev) for k in range(3)]
    g2 = _f64(dL_dmeans2D, dev).reshape(P, 3)
    gc = _f64(dL_dconic, dev).reshape(P, 4)
    gx, gy, gz = (_exact(gc[:, k], dev) for k in (0, 1, 3))
    if mutation == "conic_xy_not_halved":
        gy = gy * 0.5      # the off-diagonal conic gradient taken as the full derivative
    cov6 = [_exact(cov3D[:, k], dev) for k in range(6)]

    # ---- computeCov2DCUDA (backward.cu:141-271)
    t = _view_point(vm, p)
    tcl, passes, _ = _clamp_t(t, cam)
    x_mul, y_mul = (pa.to(torch.float64) for pa in passes)                # :172-173
    if mutation == "no_clamp_mask":
        x_mul, y_mul = torch.ones_like(x_mul), torch.ones_like(y_mul)
    T = _T(t, tcl, cam)
    V = _sym(cov6)
    TV = [[T[i][0] * V[0][j] + T[i][1] * V[1][j] + T[i][2] * V[2][j] for j in range(3)] for i in range(2)]
    a0 = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2]
    b = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2]
    c0 = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2]
    a, c = a0 + LOWPASS, c0 + LOWPASS
    denom = a * c - b * b
    d2 = denom * denom
    # det^2 + 1e-7: the reference's regulariser, visible in its outputs (:200)
    inv = 1.0 / (d2 + DET_REG) if det_reg else 1.0 / d2
    # :207-209.  dL_dconic.y arrives halved from the blend (backward.cu:545), hence 2 b c y, not b c y
    dL_da = inv * (-1.0 * c * c * gx + 2.0 * b * c * gy + (denom - a * c) * gz)
    dL_dc = inv * (-1.0 * a * a * gz + 2.0 * a * b * gy + (denom - a * c) * gx)
    dL_db = inv * 2.0 * (b * c * gx - (denom + 2.0 * b * b) * gy + a * b * gz)
    out = {}
    if antialiasing:
        # 3DGS backward.cu with antialiasing: dL/do = h g, and dL/dr = o g / (2 h) above the floor
        h, active, _ = _aa_factor(a0, b, c0)
        if mutation == "aa_h_squared":
            h = h * h
        g = _exact(_f64(dL_dopacity, dev).reshape(P), dev)
        og = _exact(_f64(opacities, dev).reshape(P), dev) * g
        out["dL_dopacity"] = g if mutation == "aa_dopacity_not_scaled" else h * g
        g_r = og / (2.0 * h)
        on = active | (mutation == "aa_cov_on_floor")
        g_r = _where(on, g_r, AV(torch.zeros_like(g_r.v)))
        dx, dz, dy = _aa_dr(a0, b, c0, mutation)
        dL_da, dL_db, dL_dc = dL_da + g_r * dx, dL_db + g_r * dz, dL_dc + g_r * dy
    # :214-224: the diagonal entries once, the off-diagonal ones doubled (each appears twice in Vrk)
    off = 1.0 if mutation == "cov_offdiag_not_doubled" else 2.0
    T0, T1 = T
    g_cov = [T0[0] * T0[0] * dL_da + T0[0] * T1[0] * dL_db + T1[0] * T1[0] * dL_dc,
             off * T0[0] * T0[1] * dL_da + (off / 2.0) * (T0[0] * T1[1] + T0[1] * T1[0]) * dL_db
             + off * T1[0] * T1[1] * dL_dc,
             off * T0[0] * T0[2] * dL_da + (off / 2.0) * (T0[0] * T1[2] + T0[2] * T1[0]) * dL_db
             + off * T1[0] * T1[2] * dL_dc,
             T0[1] * T0[1] * dL_da + T0[1] * T1[1] * dL_db + T1[1] * T1[1] * dL_dc,
             off * T0[2] * T0[1] * dL_da + (off / 2.0) * (T0[1] * T1[2] + T0[2] * T1[1]) * dL_db
             + off * T1[1] * T1[2] * dL_dc,
             T0[2] * T0[2] * dL_da + T0[2] * T1[2] * dL_db + T1[2] * T1[2] * dL_dc]
    # :234-245 dL/dT, :249-252 dL/dJ (W[col][row] = view[4 row + col])
    TVk = lambda Ti, k: Ti[0] * V[k][0] + Ti[1] * V[k][1] + Ti[2] * V[k][2]
    dT0 = [2.0 * TVk(T0, k) * dL_da + TVk(T1, k) * dL_db for k in range(3)]
    dT1 = [2.0 * TVk(T1, k) * dL_dc + TVk(T0, k) * dL_db for k in range(3)]
    Wc = lambda col: [vm[4 * r + col] for r in range(3)]
    dJ00 = sum((w * d for w, d in zip(Wc(0), dT0)), AV(torch.zeros(P, dtype=torch.float64, device=dev)))
    dJ02 = sum((w * d for w, d in zip(Wc(2), dT0)), AV(torch.zeros(P, dtype=torch.float64, device=dev)))
    dJ11 = sum((w * d for w, d in zip(Wc(1), dT1)), AV(torch.zeros(P, dtype=torch.float64, device=dev)))
    dJ12 = sum((w * d for w, d in zip(Wc(2), dT1)), AV(torch.zeros(P, dtype=torch.float64, device=dev)))
    tz = 1.0 / t[2]
    tz2 = tz * tz
    tz3 = tz2 * tz
    # :259-261.  The clamp masks only the direct tx, ty terms; dL/dtz keeps the clamped t.x, t.y
    dtx = AV(x_mul) * (-fx) * tz2 * dJ02
    dty = AV(y_mul) * (-fy) * tz2 * dJ12
    dtz = (-fx) * tz2 * dJ00 - fy * tz2 * dJ11 + (2.0 * fx * tcl[0]) * tz3 * dJ02 + (2.0 * fy * tcl[1]) * tz3 * dJ12
    # :265 transformVec4x3Transpose
    g_mean = [vm[4 * j] * dtx + vm[4 * j + 1] * dty + vm[4 * j + 2] * dtz for j in range(3)]

    # ---- projected centre (backward.cu:365-382)
    hom = _hom(pm, p)
    m_w = 1.0 / (hom[3] + W_EPS)
    mul1 = hom[0] * m_w * m_w
    mul2 = hom[1] * m_w * m_w
    gmx, gmy = _exact(g2[:, 0], dev), _exact(g2[:, 1], dev)
    for j in range(3):
        g_mean[j] = g_mean[j] + ((pm[4 * j] * m_w - pm[4 * j + 3] * mul1) * gmx
                                 + (pm[4 * j + 1] * m_w - pm[4 * j + 3] * mul2) * gmy)

    # ---- SH colour (backward.cu:20-136)
    if shs is not None:
        sh = _f64(shs, dev)
        M = sh.shape[1]
        d_orig, d = _sh_dir(means3D, cam["campos"], dev)
        x, y, z = (_col(e) for e in d)
        g_rgb = _f64(dL_dcolors, dev).reshape(P, 3)
        if mutation != "clamped_not_zeroed":
            g_rgb = torch.where(torch.as_tensor(clamped).to(dev).reshape(P, 3).bool(), torch.zeros_like(g_rgb), g_rgb)
        G = _exact(g_rgb, dev)
        S = [_exact(sh[:, k], dev) for k in range(M)]
        Y = _sh_basis(D, *d)
        sgn1 = -1.0 if mutation == "y1_sign" else 1.0
        if D > 0:
            Y[1:4] = [sgn1 * y_ for y_ in Y[1:4]]
        g_sh = [(_col(yk) * G) for yk in Y]
        zero3 = AV(torch.zeros((P, 3), dtype=torch.float64, device=dev))
        dx, dy, dz = zero3, zero3, zero3
        if D > 0:                                                        # :58-60
            dx = sgn1 * -SH_C1 * S[3]
            dy = sgn1 * -SH_C1 * S[1]
            dz = sgn1 * SH_C1 * S[2]
        if D > 1:                                                        # :78-80
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            dx = dx + SH_C2[0] * y * S[4] + SH_C2[2] * 2.0 * -x * S[6] + SH_C2[3] * z * S[7] + SH_C2[4] * 2.0 * x * S[8]
            dy = (dy + SH_C2[0] * x * S[4] + SH_C2[1] * z * S[5] + SH_C2[2] * 2.0 * -y * S[6]
                  + SH_C2[4] * 2.0 * -y * S[8])
            dz = dz + SH_C2[1] * y * S[5] + SH_C2[2] * 2.0 * 2.0 * z * S[6] + SH_C2[3] * x * S[7]
        if D > 2:                                                        # :99-119
            dx = dx + (SH_C3[0] * S[9] * 3.0 * 2.0 * xy + SH_C3[1] * S[10] * yz + SH_C3[2] * S[11] * -2.0 * xy
                       + SH_C3[3] * S[12] * -3.0 * 2.0 * xz + SH_C3[4] * S[13] * (-3.0 * xx + 4.0 * zz - yy)
                       + SH_C3[5] * S[14] * 2.0 * xz + SH_C3[6] * S[15] * 3.0 * (xx - yy))
            dy = dy + (SH_C3[0] * S[9] * 3.0 * (xx - yy) + SH_C3[1] * S[10] * xz
                       + SH_C3[2] * S[11] * (-3.0 * yy + 4.0 * zz - xx) + SH_C3[3] * S[12] * -3.0 * 2.0 * yz
                       + SH_C3[4] * S[13] * -2.0 * xy + SH_C3[5] * S[14] * -2.0 * yz
                       + SH_C3[6] * S[15] * -3.0 * 2.0 * xy)
            dz = dz + (SH_C3[1] * S[10] * xy + SH_C3[2] * S[11] * 4.0 * 2.0 * yz
                       + SH_C3[3] * S[12] * 3.0 * (2.0 * zz - xx - yy) + SH_C3[4] * S[13] * 4.0 * 2.0 * xz
                       + SH_C3[5] * S[14] * (xx - yy))
        dot3 = lambda u: u[:, 0] * G[:, 0] + u[:, 1] * G[:, 1] + u[:, 2] * G[:, 2]
        dd = [dot3(dx), dot3(dy), dot3(dz)]                               # :127
        # dnormvdv (auxiliary.h:107-117): the derivative of v / |v| at v = pos - campos
        v = d_orig
        sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2]
        invsum32 = 1.0 / (sum2 * sum2 * sum2).sqrt()
        g_dir = [((sum2 - v[0] * v[0]) * dd[0] - v[1] * v[0] * dd[1] - v[2] * v[0] * dd[2]) * invsum32,
                 (-1.0 * v[0] * v[1] * dd[0] + (sum2 - v[1] * v[1]) * dd[1] - v[2] * v[1] * dd[2]) * invsum32,
                 (-1.0 * v[0] * v[2] * dd[0] - v[1] * v[2] * dd[1] + (sum2 - v[2] * v[2]) * dd[2]) * invsum32]
        if mutation != "no_sh_direction":
            g_mean = [g_mean[j] + g_dir[j] for j in range(3)]
        n = (D + 1) ** 2
        zsh = torch.zeros((P, M, 3), dtype=torch.float64, device=dev)
        out["dL_dsh"] = AV(torch.cat([torch.stack([g.v for g in g_sh], 1), zsh[:, n:]], 1),
                           torch.cat([torch.stack([g.m for g in g_sh], 1), zsh[:, n:]], 1))

    # ---- computeCov3D backward (backward.cu:275-336)
    if scales is not None:
        s = [_exact(scales[:, k], dev) * _c(scale_modifier) for k in range(3)]   # the already-modified scale (:291)
        order = (3, 0, 1, 2) if mutation == "quat_xyzw" else (0, 1, 2, 3)
        R, (r, x, y, z) = _rotation([_exact(rotations[:, k], dev) for k in range(4)], order)   # not renormalised
        Mx = [[s[rr] * R[cc][rr] for rr in range(3)] for cc in range(3)]       # (S R)[c][r]
        # dL_dSigma: the off-diagonal gradients arrive doubled, so they are halved back (:304-307)
        h = g_cov
        dS = [[h[0], 0.5 * h[1], 0.5 * h[2]], [0.5 * h[1], h[3], 0.5 * h[4]], [0.5 * h[2], 0.5 * h[4], h[5]]]
        # dL_dM = 2 M dL_dSigma (:311): (M dS)[c][r] = sum_k M[k][r] dS[c][k]
        dM = [[2.0 * (Mx[0][rr] * dS[cc][0] + Mx[1][rr] * dS[cc][1] + Mx[2][rr] * dS[cc][2]) for rr in range(3)]
              for cc in range(3)]
        # :318-320 dL/ds_k = <Rt[k], dL_dMt[k]> = sum_r R[r][k] dM[r][k]: the gradient w.r.t. mod * scale
        g_s = [R[0][k] * dM[0][k] + R[1][k] * dM[1][k] + R[2][k] * dM[2][k] for k in range(3)]
        if mutation == "scale_times_modifier":
            g_s = [g * _c(scale_modifier) for g in g_s]
        # :322-324 dL_dMt[k][r] = s_k dM[r][k]
        Mt = [[s[k] * dM[rr][k] for rr in range(3)] for k in range(3)]
        gq = [2.0 * z * (Mt[0][1] - Mt[1][0]) + 2.0 * y * (Mt[2][0] - Mt[0][2]) + 2.0 * x * (Mt[1][2] - Mt[2][1]),
              2.0 * y * (Mt[1][0] + Mt[0][1]) + 2.0 * z * (Mt[2][0] + Mt[0][2]) + 2.0 * r * (Mt[1][2] - Mt[2][1])
              - 4.0 * x * (Mt[2][2] + Mt[1][1]),
              2.0 * x * (Mt[1][0] + Mt[0][1]) + 2.0 * r * (Mt[2][0] - Mt[0][2]) + 2.0 * z * (Mt[1][2] + Mt[2][1])
              - 4.0 * y * (Mt[2][2] + Mt[0][0]),
              2.0 * r * (Mt[0][1] - Mt[1][0]) + 2.0 * x * (Mt[2][0] + Mt[0][2]) + 2.0 * y * (Mt[1][2] + Mt[2][1])
              - 4.0 * z * (Mt[1][1] + Mt[0][0])]                          # :328-331, written as given (:335)
        if mutation == "quat_xyzw":   # written back in the order it was misread
            gq = [gq[1], gq[2], gq[3], gq[0]]
        out["dL_dscales"] = stack(g_s)
        out["dL_drotations"] = stack(gq)

    out["dL_dmeans3D"] = stack(g_mean)
    out["dL_dcov3D"] = stack(g_cov)
    keep = torch.as_tensor(radii).to(dev).reshape(-1) > 0                 # :153, :362: culled Gaussians stay zero
    for k, a_ in out.items():
        sel = keep.reshape((P,) + (1,) * (a_.v.dim() - 1))
        out[k] = AV(torch.where(sel, a_.v, torch.zeros_like(a_.v)), torch.where(sel, a_.m, torch.zeros_like(a_.m)))
    return out


def compare(got, want: AV, mask=None, rtol=RTOL) -> float:
    """max over entries (of the Gaussians in mask) of |got - want| / (rtol * magnitude): <= 1 passes.  An entry of
    magnitude 0 (a culled Gaussian, an SH coefficient above the active degree) must be exactly equal.  There is no
    allowance for a fraction of bad entries."""
    g = torch.as_tensor(got).detach().to(dtype=torch.float64, device=want.v.device).reshape(want.v.shape)
    diff = (g - want.v).abs()
    if mask is not None:
        m = torch.as_tensor(mask).to(want.v.device).reshape((-1,) + (1,) * (diff.dim() - 1)).expand_as(diff)
        diff, mag = diff[m], want.m[m]
    else:
        mag = want.m
    if diff.numel() == 0:
        return 0.0
    if not bool(torch.isfinite(diff).all()):
        return float("inf")
    r = torch.where(diff == 0, torch.zeros_like(diff), diff / (rtol * mag))   # diff > 0 = magnitude: inf
    return float(r.max())
