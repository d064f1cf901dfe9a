"""TEST INFRASTRUCTURE ONLY — numpy float64 statement of one Adam step with a row mask, the checker for
semantic-gaussians_b200/csrc/adam.cu and semantic-gaussians_b200/optim.py (never imported by the product path).

torch.optim.Adam without amsgrad / weight_decay / maximize at global step t (1-based):

    m = m + (g - m) (1 - beta1)        v = beta2 v + (1 - beta2) g^2
    p = p - lr / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)

applied to the rows where ``visible`` is set (all rows when it is None); every other row is returned unchanged."""
import numpy as np


def adam_step(p, g, m, v, t, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, visible=None):
    """(p, m, v) after step t, float64, from the state before it (any float dtype, first axis = rows).  The gradient
    of a row that is not visible is not read (it may be NaN)."""
    p, m, v = (np.array(a, dtype=np.float64) for a in (p, m, v))
    rows = slice(None) if visible is None else np.asarray(visible).astype(bool)
    beta1, beta2 = float(betas[0]), float(betas[1])
    gr = np.asarray(g, dtype=np.float64)[rows]
    mr = m[rows] + (gr - m[rows]) * (1.0 - beta1)
    vr = beta2 * v[rows] + (1.0 - beta2) * gr * gr
    step_size = lr / (1.0 - beta1 ** t)
    p[rows] = p[rows] - step_size * (mr / (np.sqrt(vr) / np.sqrt(1.0 - beta2 ** t) + eps))
    m[rows] = mr
    v[rows] = vr
    return p, m, v
