"""Scene recipes that push Gaussians onto the geometry stage's branches (numpy only, no GPU): view-space
placement relative to a SynthCamera and the sideways push beyond the 1.3 tan(fov / 2) frustum clamp."""
import math

import numpy as np


def view_space(scene, cam):
    """(P, 3) float64 view-space centres t = p @ view[:3, :3] + view[3, :3] (row-vector convention)."""
    view = np.asarray(cam.world_view_transform, np.float64).reshape(4, 4)
    return scene.xyz.astype(np.float64) @ view[:3, :3] + view[3, :3], view


def set_view_space(scene, t, view, sel):
    """Move the Gaussians in sel to view-space centres t[sel]."""
    xyz = (t - view[3, :3]) @ np.linalg.inv(view[:3, :3])
    scene.xyz[sel] = xyz[sel].astype(np.float32)


def push_sideways(scene, cam, axes, every=10, factor=1.45, grow=8.0):
    """Every `every`-th Gaussian moved sideways in view space to |t_k / t_z| = factor tan(fov / 2), beyond the
    1.3 tan(fov / 2) clamp, on the given axes ("x", "y" or both), keeping its depth, and made `grow` times larger
    so that it still reaches the image (the recipe of test_geom_grad_cpu.py's clamp test).  Returns the selection."""
    t, view = view_space(scene, cam)
    sel = np.arange(scene.P) % every == 0
    for ax in axes:
        k, tan = (0, math.tan(cam.FoVx * 0.5)) if ax == "x" else (1, math.tan(cam.FoVy * 0.5))
        t[sel, k] = np.sign(t[sel, k] + 1e-9) * factor * tan * np.abs(t[sel, 2])
    scene.scales[sel] *= grow
    set_view_space(scene, t, view, sel)
    return sel
