"""Float64 restatement of the sparse convolution (sparse.py) and MinkUNet (mink_unet.py) for the tests.

Coordinate maps and kernel maps are built with Python dicts over coordinate tuples; the products are float64 torch
expressions on the CPU (gather, matmul, index_add_), so autograd gives the reference gradients.  Orders are the ones
sgb200.h documents: a strided map lists its rows in the order their first child appears, and an offset's pairs ascend
in the output row."""
from __future__ import annotations

import torch
import torch.nn.functional as Fn


def offsets(k, t):
    """Kernel offsets (dx, dy, dz) by index d = jx + k jy + k^2 jz, per axis lb + j t with lb = -((k-1)//2) t."""
    lb = -((k - 1) // 2) * t
    return [(lb + jx * t, lb + jy * t, lb + jz * t) for jz in range(k) for jy in range(k) for jx in range(k)]


def stride_map(rows, t):
    """Rows (b, x, y, z) at stride 2t from rows at stride t: unique parents in order of first appearance."""
    t2, seen, out = 2 * t, set(), []
    for b, x, y, z in rows:
        p = (b, x // t2 * t2, y // t2 * t2, z // t2 * t2)
        if p not in seen:
            seen.add(p)
            out.append(p)
    return out


def kernel_map(in_rows, out_rows, k, t):
    """Per offset, the (in row, out row) pairs with in = out + offset and equal b, ascending in the out row."""
    index = {tuple(r): i for i, r in enumerate(in_rows)}
    maps = []
    for dx, dy, dz in offsets(k, t):
        maps.append([(index[q], o) for o, q in ((o, (b, x + dx, y + dy, z + dz)) for o, (b, x, y, z) in enumerate(out_rows))
                     if q in index])
    return maps


def conv(x, W, kmap, n_out, transposed=False):
    """sum over offsets of gathered products: out[o] += x[i] W_d, or with the roles swapped for a transposed layer."""
    out = torch.zeros((n_out, W.shape[-1]), dtype=x.dtype)
    for d, pairs in enumerate(kmap):
        if not pairs:
            continue
        p = torch.tensor(pairs, dtype=torch.int64)
        src, dst = (p[:, 1], p[:, 0]) if transposed else (p[:, 0], p[:, 1])
        out = out.index_add(0, dst, x[src] @ W[d])
    return out


class Maps:
    """The restatement of CoordinateManager: rows by stride and kernel maps by (in stride, out stride, k)."""

    def __init__(self, rows):
        self.rows = {1: [tuple(r) for r in rows]}
        self.kmaps = {}

    def at(self, t):
        if t not in self.rows:
            self.rows[t] = stride_map(self.at(t // 2), t // 2)
        return self.rows[t]

    def kmap(self, t_in, t_out, k):
        key = (t_in, t_out, k)
        if key not in self.kmaps:
            self.kmaps[key] = kernel_map(self.at(t_in), self.at(t_out), k, t_in)
        return self.kmaps[key]


def minkunet_forward(model, coords, feats, params, training):
    """MinkUNetBase.forward on the CPU in the dtype of ``feats`` (float64 for the reference values).  ``params``:
    name -> leaf tensor of that dtype for every parameter of ``model`` (buffers are read from the model).  Returns the
    output features (N, C_out)."""
    from semantic_gaussians_b200 import sparse as sp
    from semantic_gaussians_b200.mink_unet import BasicBlock

    maps = Maps(coords.tolist())
    names = {m: n for n, m in model.named_modules()}

    def P(mod, leaf):
        return params[f"{names[mod]}.{leaf}" if names[mod] else leaf]

    def run(mod, x):
        F, t = x
        if isinstance(mod, sp.Convolution):
            if mod.kernel_size == 1:
                return F @ P(mod, "kernel"), t
            to = t * mod.stride
            return conv(F, P(mod, "kernel"), maps.kmap(t, to, mod.kernel_size), len(maps.at(to))), to
        if isinstance(mod, sp.ConvolutionTranspose):
            to = t // 2
            return conv(F, P(mod, "kernel"), maps.kmap(to, t, 2), len(maps.at(to)), transposed=True), to
        if isinstance(mod, sp.BatchNorm):
            bn = mod.bn
            return Fn.batch_norm(F, bn.running_mean.detach().cpu().to(F.dtype), bn.running_var.detach().cpu().to(F.dtype),
                                 P(bn, "weight"), P(bn, "bias"), training, bn.momentum, bn.eps), t
        if isinstance(mod, sp.ReLU):
            return torch.relu(F), t
        if isinstance(mod, torch.nn.Sequential):
            for m in mod:
                x = run(m, x)
            return x
        if isinstance(mod, BasicBlock):
            out = run(mod.relu, run(mod.norm1, run(mod.conv1, x)))
            out = run(mod.norm2, run(mod.conv2, out))
            res = run(mod.downsample, x) if mod.downsample is not None else x
            return torch.relu(out[0] + res[0]), t
        raise TypeError(type(mod))

    def cbr(conv_, bn, x):
        return run(model.relu, run(bn, run(conv_, x)))

    def cat(a, b):
        assert a[1] == b[1]
        return torch.cat([a[0], b[0]], dim=1), a[1]

    m = model
    out_p1 = cbr(m.conv0p1s1, m.bn0, (feats, 1))
    out_b1p2 = run(m.block1, cbr(m.conv1p1s2, m.bn1, out_p1))
    out_b2p4 = run(m.block2, cbr(m.conv2p2s2, m.bn2, out_b1p2))
    out_b3p8 = run(m.block3, cbr(m.conv3p4s2, m.bn3, out_b2p4))
    out = run(m.block4, cbr(m.conv4p8s2, m.bn4, out_b3p8))
    out = run(m.block5, cat(cbr(m.convtr4p16s2, m.bntr4, out), out_b3p8))
    out = run(m.block6, cat(cbr(m.convtr5p8s2, m.bntr5, out), out_b2p4))
    out = run(m.block7, cat(cbr(m.convtr6p4s2, m.bntr6, out), out_b1p2))
    out = run(m.block8, cat(cbr(m.convtr7p2s2, m.bntr7, out), out_p1))
    return run(m.final, out)[0]
