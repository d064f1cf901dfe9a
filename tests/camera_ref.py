"""The camera gradient of the geometry stage restated in float64 for the tests, by automatic differentiation.

The forward is written out here in float64 torch (view-space centre, frustum-clamped perspective Jacobian, screen
covariance, projected centre, view-space depth, SH colour through sh_utils.eval_sh) with the camera tensors expanded
to one copy per Gaussian, so that ONE backward of the surrogate loss

    L = sum_i <G_C,i, C_i> + g_ndc,i . ndc_i + gz_i z_i + g_rgb,i . rgb_i

gives every Gaussian's own contribution to dL/dviewmatrix, dL/dprojmatrix and dL/dcampos (rows of the copies).  The
upstream gradients are the kernel's own inputs: dL_dmeans2D (NDC units), dL_dconic (x, y, _, w) with the xy entry
halved as the blend writes it, dL_dcolors masked where the forward clamped, dL/dz.  G_C = dL/dC is autograd's
gradient of the conic K = C^-1 scaled by det^2 / (det^2 + 1e-7), the reference's regulariser (geom_ref.DET_REG).
Conventions held as the forward holds them: where the Jacobian's evaluation point is clamped sideways, the clamped
t_x (t_y) is a constant; focal lengths are fp32 constants.

With antialiasing a fifth path is the opacity factor: L_aa = sum_i g_i o_i h_i(C0_i) with g = dL/d(o h) the blend's
opacity gradient (what the geometry kernel reads before it overwrites dL_dopacity with h g), o the raw opacity and
h = sqrt(max(2.5e-5, det C0 / det C)) of the undilated screen covariance C0 = C - 0.3 I; on the floor h is constant.
Which side of the floor a Gaussian is on is the kernel's fp32 decision (the sign of the h it stored, aa_active), not
a float64 one: where det C0 / det C lies within rounding of the floor the two could differ, and the whole term of
that Gaussian would count as error (geom_ref's comparison checks that decision, leaving out its fragile band).

Magnitude: per Gaussian and entry, mag = kappa |c_cov| + |c_ndc| + |c_z| + |c_rgb| (+ kappa0 |c_aa|) from separate
backwards (one per path), kappa the screen covariance's conditioning (geom_ref) and kappa0 that of C0, whose
determinant h is formed from.  A per-view camera gradient passes when |got - sum_i c_i| <= RTOL * sum_i mag_i entry
by entry.
"""
from __future__ import annotations

import numpy as np
import torch

from geom_ref import AA_FLOOR, DET_REG, EPS32, LOWPASS, W_EPS, _c

from semantic_gaussians_b200.sh_utils import eval_sh

# Tolerance factor of the per-view sums: geom_ref.RTOL's 16 * 2^-24.  The host build of geom_grad.cuh stays within
# 0.05 RTOL on the CPU cases of test_camera_grad_cpu.py (twenty times below it); every family of
# test_camera_grad_gpu.py passes within it on an H100 80GB HBM3 at a 700 W power limit.
RTOL = 16 * EPS32

NEVER_READ_VIEW = (3, 7, 11, 15)
NEVER_READ_PROJ = (2, 6, 10, 14)


def _f64(a, dev):
    return torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(dev, torch.float64)


def camera_terms(means3D, radii, cov3D, view, proj, campos, W, H, tan_fovx, tan_fovy, dL_dmeans2D, dL_dconic, *,
                 shs=None, D=0, clamped=None, dL_dcolors=None, dL_ddepth=None, antialiasing=False, opacities=None,
                 dL_dopacity=None, aa_active=None, dev="cpu"):
    """Per-Gaussian camera-gradient contributions (P, 35) = [dview 16 | dproj 16 | dcampos 3] (element order of the
    flattened fp32 camera arrays the kernel reads) and their magnitudes (P, 35), both float64; culled Gaussians
    (radii <= 0) get zeros.  antialiasing: opacities (P,) the raw o, dL_dopacity (P,) the blend's g = dL/d(o h),
    aa_active (P,) the branch the kernel took (h > 0: above the floor)."""
    assert not antialiasing or all(x is not None for x in (opacities, dL_dopacity, aa_active))
    P = int(np.asarray(radii.cpu() if isinstance(radii, torch.Tensor) else radii).shape[0])
    keep = torch.as_tensor(np.asarray(radii.cpu() if isinstance(radii, torch.Tensor) else radii)).reshape(-1) > 0
    idx = torch.nonzero(keep).reshape(-1).to(dev)
    n = idx.numel()
    pick = lambda a, w: _f64(a, dev).reshape(P, w)[idx]  # noqa: E731
    p = pick(means3D, 3)
    cov = pick(cov3D, 6)
    g2 = pick(dL_dmeans2D, 3)
    gc = pick(dL_dconic, 4)
    view0 = _f64(np.asarray(view, np.float32).reshape(-1), dev)
    proj0 = _f64(np.asarray(proj, np.float32).reshape(-1), dev)
    cpos0 = _f64(np.asarray(campos, np.float32).reshape(-1), dev)
    tx32, ty32 = np.float32(tan_fovx), np.float32(tan_fovy)
    fx = float(np.float32(W) / (np.float32(2.0) * tx32))
    fy = float(np.float32(H) / (np.float32(2.0) * ty32))
    limx, limy = _c(np.float32(1.3) * tx32), _c(np.float32(1.3) * ty32)

    def forward(vm, pm, cp):
        """The four loss paths, each summed over the Gaussians."""
        Wm = lambda i, j: vm[:, 4 * j + i]  # noqa: E731
        t = [Wm(i, 0) * p[:, 0] + Wm(i, 1) * p[:, 1] + Wm(i, 2) * p[:, 2] + vm[:, 12 + i] for i in range(3)]
        tz = t[2]
        tcl = []
        for k, lim in ((0, limx), (1, limy)):
            r = t[k] / tz
            inside = ((r >= -lim) & (r <= lim)).detach()
            tcl.append(torch.where(inside, t[k], (r.clamp(-lim, lim) * tz).detach()))
        J00, J02 = fx / tz, -fx * tcl[0] / (tz * tz)
        J11, J12 = fy / tz, -fy * tcl[1] / (tz * tz)
        A0 = torch.stack([J00 * Wm(0, j) + J02 * Wm(2, j) for j in range(3)], 1)
        A1 = torch.stack([J11 * Wm(1, j) + J12 * Wm(2, j) for j in range(3)], 1)
        S = torch.stack([cov[:, [0, 1, 2]], cov[:, [1, 3, 4]], cov[:, [2, 4, 5]]], 1)
        A = torch.stack([A0, A1], 1)                                   # (n, 2, 3)
        Cm = A @ S @ A.transpose(1, 2) + LOWPASS * torch.eye(2, dtype=torch.float64, device=dev)
        # dL/dC: autograd of the conic loss through the inverse, with the reference's det^2 regulariser
        with torch.enable_grad():
            Cd = Cm.detach().requires_grad_(True)
            K = torch.linalg.inv(Cd)
            lk = (gc[:, 0] * K[:, 0, 0] + 2.0 * gc[:, 1] * K[:, 0, 1] + gc[:, 3] * K[:, 1, 1]).sum()
            (G,) = torch.autograd.grad(lk, Cd)
            det = torch.linalg.det(Cd.detach())
            G = G * (det * det / (det * det + DET_REG))[:, None, None]
        l_cov = (G.detach() * Cm).sum()
        hom = [pm[:, k] * p[:, 0] + pm[:, 4 + k] * p[:, 1] + pm[:, 8 + k] * p[:, 2] + pm[:, 12 + k] for k in range(4)]
        iw = 1.0 / (hom[3] + W_EPS)
        l_ndc = (g2[:, 0] * hom[0] * iw + g2[:, 1] * hom[1] * iw).sum()
        l_z = (pick(dL_ddepth, 1)[:, 0] * tz).sum() if dL_ddepth is not None else tz.sum() * 0.0
        if shs is not None:
            sh = _f64(shs, dev).reshape(P, -1, 3)[idx]
            v = p - cp
            d = v / v.norm(dim=1, keepdim=True)
            rgb = eval_sh(D, sh.transpose(1, 2), d) + 0.5
            g = pick(dL_dcolors, 3) * (~torch.as_tensor(np.asarray(clamped.cpu() if isinstance(clamped, torch.Tensor)
                                                                   else clamped)).reshape(P, 3)[idx.cpu()].bool()
                                       ).to(dev, torch.float64)
            l_rgb = (g * rgb).sum()
        else:
            l_rgb = tz.sum() * 0.0
        l_aa = tz.sum() * 0.0
        if antialiasing:
            C0 = Cm - LOWPASS * torch.eye(2, dtype=torch.float64, device=dev)
            r = torch.linalg.det(C0) / torch.linalg.det(Cm)
            active = pick(aa_active, 1)[:, 0] > 0
            # the floor branch is constant: no camera gradient
            h = torch.where(active, r.clamp(min=1e-300).sqrt(), torch.full_like(r, AA_FLOOR ** 0.5))
            l_aa = (pick(opacities, 1)[:, 0] * pick(dL_dopacity, 1)[:, 0] * h).sum()
        return l_cov, l_ndc, l_z, l_rgb, l_aa, Cm.detach()

    vm = view0.expand(n, 16).clone().requires_grad_(True)
    pm = proj0.expand(n, 16).clone().requires_grad_(True)
    cp = cpos0.expand(n, 3).clone().requires_grad_(True)
    with torch.enable_grad():
        losses = forward(vm, pm, cp)
        parts = []
        for loss in losses[:5]:
            gs = (torch.autograd.grad(loss, (vm, pm, cp), retain_graph=True, allow_unused=True) if loss.requires_grad
                  else (None, None, None))   # SH degree 0: the colour does not depend on the camera
            parts.append(torch.cat([torch.zeros((n, w), dtype=torch.float64, device=dev) if g is None else g
                                    for g, w in zip(gs, (16, 16, 3))], 1))
    Cm = losses[5]
    a, b, c = Cm[:, 0, 0], Cm[:, 0, 1], Cm[:, 1, 1]
    kappa = ((a * c).abs() + b * b) / (a * c - b * b).abs()
    a0, c0 = a - LOWPASS, c - LOWPASS
    kappa0 = ((a0 * c0).abs() + b * b) / (a0 * c0 - b * b).abs()
    contrib = parts[0] + parts[1] + parts[2] + parts[3] + parts[4]
    mag = (kappa[:, None] * parts[0].abs() + parts[1].abs() + parts[2].abs() + parts[3].abs()
           + torch.where(parts[4] == 0, torch.zeros_like(parts[4]), kappa0[:, None] * parts[4].abs()))
    full = torch.zeros((P, 35), dtype=torch.float64, device=dev)
    fmag = torch.zeros((P, 35), dtype=torch.float64, device=dev)
    full[idx], fmag[idx] = contrib, mag
    return full, fmag


def check_sum(got35, contrib, mag, rtol=RTOL) -> float:
    """max over the 35 entries of |got - sum_i c_i| / (rtol * sum_i mag_i) (<= 1 passes); the entries the forward
    never reads must be exactly 0 (returns inf otherwise)."""
    got = torch.as_tensor(got35).to(torch.float64).reshape(35).cpu()
    want, m = contrib.sum(0).cpu(), mag.sum(0).cpu()
    zero = list(NEVER_READ_VIEW) + [16 + k for k in NEVER_READ_PROJ]
    if bool((got[zero] != 0).any()) or not bool(torch.isfinite(got).all()):
        return float("inf")
    live = [k for k in range(35) if k not in zero]
    diff = (got[live] - want[live]).abs()
    den = rtol * m[live]
    r = torch.where(diff == 0, torch.zeros_like(diff), diff / den)
    return float(r.max())
