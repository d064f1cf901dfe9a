"""Float64 restatement of the sparse convolution (sparse.py) and MinkUNet (mink_unet.py) for the tests.

Coordinate maps and kernel maps are built twice, neither way sharing logic with the device hash table: with Python
dicts over coordinate tuples (Maps, for hand-checkable sizes), and with sorting torch expressions on any device
(TensorMaps, for maps of a million rows).  The products are float64 torch expressions on the inputs' device (gather,
matmul, index_add_), so autograd gives the reference gradients.  Orders are the ones sgb200.h documents: a strided map
lists its rows in the order their first child appears, and an offset's pairs ascend in the output row.

``random_rows`` draws the (b, x, y, z) test clouds of the GPU tests."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as Fn


def random_rows(kind, N, batches, seed=0):
    """N distinct int32 rows (b, x, y, z) in random order, b < batches.  Kinds: "box", a cube at ~30 % occupancy;
    "near_2_30", coordinates just below 2^30; "low_bits", coordinates that differ only in bit 0 and above bit 20."""
    rng = np.random.default_rng(seed)
    if kind == "box":
        side = max(4, int(round((N / batches / 0.3) ** (1 / 3))))        # ~30 % occupancy
        pts = rng.integers(0, side, (3 * N, 3))
    elif kind == "near_2_30":
        pts = (1 << 30) - 1024 + rng.integers(0, 64, (3 * N, 3)) * 32 + rng.integers(0, 3, (3 * N, 3))
    else:   # low_bits: rows that differ only above bit 20
        pts = (rng.integers(0, 64, (3 * N, 3)) << 20) + rng.integers(0, 2, (3 * N, 3))
    b = rng.integers(0, batches, (3 * N, 1))
    out = np.unique(np.concatenate([b, pts], 1), axis=0)
    out = out[rng.permutation(len(out))[:N]]
    assert len(out) == N
    return out.astype(np.int32)


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
    """sum over offsets of gathered products: out[o] += x[i] W_d, or with the roles swapped for a transposed layer.
    ``kmap``: per offset, the (in row, out row) pairs as a list of tuples or an (n, 2) tensor; computed on x's device."""
    out = torch.zeros((n_out, W.shape[-1]), dtype=x.dtype, device=x.device)
    for d, pairs in enumerate(kmap):
        if len(pairs) == 0:
            continue
        p = torch.as_tensor(pairs, dtype=torch.int64, device=x.device)
        src, dst = (p[:, 1], p[:, 0]) if transposed else (p[:, 0], p[:, 1])
        out = out.index_add(0, dst, x[src] @ W[d])
    return out


# (in stride, out stride, k) of every kernel map MinkUNet builds
MINKUNET_KMAPS = [(1, 1, 5)] + [(t, t, 3) for t in (1, 2, 4, 8, 16)] + [(t, 2 * t, 2) for t in (1, 2, 4, 8)]


class Maps:
    """The restatement of CoordinateManager: rows by stride and kernel maps by (in stride, out stride, k)."""
    stride_map = staticmethod(stride_map)
    kernel_map = staticmethod(kernel_map)

    def __init__(self, rows):
        self.rows = {1: [tuple(r) for r in rows]}
        self.kmaps = {}

    def at(self, t):
        if t not in self.rows:
            self.rows[t] = self.stride_map(self.at(t // 2), t // 2)
        return self.rows[t]

    def kmap(self, t_in, t_out, k):
        key = (t_in, t_out, k)
        if key not in self.kmaps:
            self.kmaps[key] = self.kernel_map(self.at(t_in), self.at(t_out), k, t_in)
        return self.kmaps[key]


# ---------------------------------------------------------------- the same maps as torch expressions

def stride_map_t(rows, t):
    """stride_map on an (N, 4) integer tensor: the parents by floor, unique, in order of their first child's row."""
    r = rows.long()
    t2 = 2 * t
    par = torch.cat([r[:, :1], torch.div(r[:, 1:], t2, rounding_mode="floor") * t2], 1)
    uniq, inv = torch.unique(par, dim=0, return_inverse=True)
    first = torch.full((len(uniq),), len(r), dtype=torch.int64, device=r.device)
    first = first.scatter_reduce(0, inv, torch.arange(len(r), device=r.device), "amin")
    return uniq[first.argsort()].to(rows.dtype)


class RowIndex:
    """Row lookup in a set of (b, x, y, z) rows by sorting.  Each component is replaced by its rank among the set's
    values of that component (torch.unique, so any int32 values, such as the "low_bits" rows, work), and the four
    ranks are packed mixed-radix into one int64 key; the set's keys are sorted and queries found by searchsorted."""

    def __init__(self, rows):
        r = rows.long()
        self.values = [torch.unique(r[:, a]) for a in range(4)]
        assert math.prod(len(v) for v in self.values) < 2 ** 62, "rows too varied to pack into one int64 key"
        key, _ = self._key(r)
        self.keys, self.order = key.sort()

    def _key(self, r):
        """(key, known): known is False where a component is not among the set's values (the key is then junk)."""
        key = torch.zeros(len(r), dtype=torch.int64, device=r.device)
        known = torch.ones(len(r), dtype=torch.bool, device=r.device)
        for a, v in enumerate(self.values):
            c = r[:, a].contiguous()
            pos = torch.searchsorted(v, c).clamp_max(len(v) - 1)
            known &= v[pos] == c
            key = key * len(v) + pos
        return key, known

    def find(self, queries):
        """Row of the set equal to each query row (int64, any values), or -1."""
        key, known = self._key(queries)
        pos = torch.searchsorted(self.keys, key).clamp_max(len(self.keys) - 1)
        return torch.where(known & (self.keys[pos] == key), self.order[pos], -1)


def kernel_map_t(in_rows, out_rows, k, t):
    """kernel_map on tensors: per offset an (n, 2) int64 tensor of (in row, out row) pairs, ascending in the out row."""
    index = RowIndex(in_rows)
    out = out_rows.long()
    maps = []
    for off in offsets(k, t):
        i = index.find(out + torch.tensor((0,) + off, device=out.device))
        o = torch.nonzero(i >= 0).squeeze(1)
        maps.append(torch.stack([i[o], o], 1))
    return maps


class TensorMaps(Maps):
    """Maps over an (N, 4) integer tensor: rows by stride as tensors, kernel maps as per-offset pair tensors."""
    stride_map = staticmethod(stride_map_t)
    kernel_map = staticmethod(kernel_map_t)

    def __init__(self, rows):
        self.rows = {1: rows}
        self.kmaps = {}


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
