"""Shared by test_adam_cpu.py / test_adam_gpu.py: compare one optimizer step with oracle/adam_oracle.py."""
import numpy as np

from oracle.adam_oracle import adam_step


def assert_step_matches_oracle(before, after, t, lr, betas, eps, visible=None, rtol=2e-6):
    """before = (p, g, m, v) and after = (p, m, v) as fp32 numpy arrays, first axis = rows.  The oracle is fed the fp32
    state the step started from, so only this step's rounding is compared.

    Rows that are not visible must be bitwise unchanged.  On visible rows v has no cancellation and is held to rtol
    alone (atol 1e-30 near 0).  m = m0 + (g - m0)(1 - beta1) can cancel, so its error is bounded by rtol of its operands'
    magnitude |m0| + |g|, and the error of p by rtol of the update those operands would give, plus the rounding of p
    itself (half an ulp)."""
    p0, g, m0, v0 = before
    p1, m1, v1 = after
    rows = np.ones(p0.shape[0], bool) if visible is None else np.asarray(visible).astype(bool)
    for a0, a1, name in ((p0, p1, "p"), (m0, m1, "m"), (v0, v1, "v")):
        assert np.array_equal(a0[~rows].view(np.uint32), a1[~rows].view(np.uint32)), f"{name}: a masked row changed"
    wp, wm, wv = adam_step(p0, g, m0, v0, t, lr=lr, betas=betas, eps=eps, visible=rows)
    g64, m64 = g[rows].astype(np.float64), m0[rows].astype(np.float64)
    assert np.isfinite(p1[rows]).all() and np.isfinite(m1[rows]).all() and np.isfinite(v1[rows]).all()

    def within(name, got, want, tol):
        excess = np.abs(got - want) / tol
        assert (excess <= 1.0).all(), f"{name}: error {float(excess.max()):.3g} x its tolerance"

    within("v", v1[rows], wv[rows], rtol * np.abs(wv[rows]) + 1e-30)
    within("m", m1[rows], wm[rows], rtol * (np.abs(m64) + np.abs(g64)) + 1e-30)
    scale = lr / (1.0 - betas[0] ** t) * (np.abs(m64) + np.abs(g64)) / (np.sqrt(wv[rows]) / np.sqrt(1.0 - betas[1] ** t) + eps)
    within("p", p1[rows], wp[rows], rtol * scale + 2.0 ** -23 * np.abs(wp[rows]) + 1e-30)
