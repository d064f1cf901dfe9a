"""Sparse 3D convolution and MinkUNet without a GPU: the float64 restatement against hand-worked cases, its tensor maps
against its dict maps, the MinkUNet state_dict against the reference's layer structure, and argument validation before
any CUDA call."""
import ctypes as C

import numpy as np
import pytest
import torch

import sparse_ref as ref
from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200 import sparse as sp
from semantic_gaussians_b200.mink_unet import ARCHS, mink_unet


# ---------------------------------------------------------------- the restatement, by hand

def test_stride_two_parent_of_every_point():
    rows = [(0, x, y, z) for x in range(4) for y in range(4) for z in range(4)]
    par = ref.stride_map(rows, 1)
    assert len(par) == 8 and par[0] == (0, 0, 0, 0) and par[1] == (0, 0, 0, 2)
    km = ref.kernel_map(rows, par, 2, 1)
    assert [len(p) for p in km] == [8] * 8
    for o, (b, px, py, pz) in enumerate(par):
        children = sorted(i for pairs in km for i, oo in pairs if oo == o)
        assert [rows[i] for i in children] == sorted((b, px + dx, py + dy, pz + dz)
                                                     for dx in (0, 1) for dy in (0, 1) for dz in (0, 1))
    assert ref.stride_map([(0, 6, 4, 12)], 2) == [(0, 4, 4, 12)]       # floor(c / 4) * 4
    assert ref.stride_map([(0, 7, 3, 8), (0, 5, 0, 9), (1, 4, 0, 8)], 2) == [(0, 4, 0, 8), (1, 4, 0, 8)]


@pytest.mark.parametrize("k,t", [(3, 1), (3, 4), (5, 1), (5, 2), (2, 1), (2, 8)])
def test_offset_index_of_every_offset(k, t):
    offs = ref.offsets(k, t)
    assert len(offs) == k ** 3 and len(set(offs)) == k ** 3
    lb = 0 if k == 2 else -((k - 1) // 2) * t
    for d, (dx, dy, dz) in enumerate(offs):
        jx, jy, jz = d % k, d // k % k, d // (k * k)
        assert (dx, dy, dz) == (lb + jx * t, lb + jy * t, lb + jz * t)
    if k == 3:
        assert offs[0] == (-t, -t, -t) and offs[1] == (0, -t, -t) and offs[3] == (-t, 0, -t) and offs[9] == (-t, -t, 0)
        assert offs[13] == (0, 0, 0) and offs[26] == (t, t, t)
    if k == 5:
        assert offs[0] == (-2 * t,) * 3 and offs[62] == (0, 0, 0) and offs[124] == (2 * t,) * 3
        assert offs[5] == (-2 * t, -t, -2 * t)
    if k == 2:
        assert offs == [(0, 0, 0), (t, 0, 0), (0, t, 0), (t, t, 0), (0, 0, t), (t, 0, t), (0, t, t), (t, t, t)]


def test_transposed_layer_writes_each_fine_row_from_one_coarse_row():
    fine = [(0, 0, 0, 0), (0, 1, 0, 0), (0, 1, 1, 1), (0, 2, 0, 0), (0, 3, 3, 3)]
    coarse = ref.stride_map(fine, 1)
    km = ref.kernel_map(fine, coarse, 2, 1)
    n_out = len(coarse)
    x = torch.arange(1, n_out + 1, dtype=torch.float64).reshape(n_out, 1)     # coarse row r carries r + 1
    W = torch.stack([torch.full((1, 1), 10.0 ** d, dtype=torch.float64) for d in range(8)])
    y = ref.conv(x, W, km, len(fine), transposed=True)
    # fine (0,1,1,1) is coarse (0,0,0,0) at offset (1,1,1) = index 7; fine (0,3,3,3) is coarse 2 at index 7
    assert y.flatten().tolist() == [1.0, 10.0, 1e7, 2.0, 3e7]


def test_rows_that_differ_only_in_b_never_pair():
    rows = [(0, 2, 2, 2), (1, 2, 2, 2), (1, 3, 2, 2), (2, 2, 3, 2)]
    km = ref.kernel_map(rows, rows, 3, 1)
    for d, pairs in enumerate(km):
        for i, o in pairs:
            assert rows[i][0] == rows[o][0]
    assert sum(len(p) for p in km) == 4 + 2        # 4 centres, (1,3,2,2) <-> (1,2,2,2) both ways
    assert ref.stride_map(rows, 1) == [(0, 2, 2, 2), (1, 2, 2, 2)] + [(2, 2, 2, 2)]


# ---------------------------------------------------------------- the tensor maps against the dict maps

def _cloud(kind, N, batches):
    if kind == "copies":      # one box cloud in every batch: rows that differ only in b
        base = ref.random_rows("box", N // batches, 1, seed=N)
        return np.concatenate([np.concatenate([np.full((len(base), 1), b, np.int32), base[:, 1:]], 1)
                               for b in range(batches)])
    return ref.random_rows(kind, N, batches, seed=N)


@pytest.mark.parametrize("kind,N,batches", [("box", 1, 1), ("box", 2, 1), ("box", 2, 2), ("box", 300, 1),
                                            ("box", 700, 3), ("box", 2000, 4), ("copies", 2, 2), ("copies", 800, 4),
                                            ("low_bits", 500, 2), ("near_2_30", 500, 3)])
def test_tensor_maps_equal_the_dict_maps(kind, N, batches):
    rows = _cloud(kind, N, batches)
    maps, tmaps = ref.Maps(rows.tolist()), ref.TensorMaps(torch.from_numpy(rows))
    for t in (1, 2, 4, 8, 16):
        got = tmaps.at(t)
        assert got.dtype == torch.int32 and [tuple(r) for r in got.tolist()] == maps.at(t), t
    for t_in, t_out, k in ref.MINKUNET_KMAPS:
        got = tmaps.kmap(t_in, t_out, k)
        assert len(got) == k ** 3
        assert [[tuple(p) for p in pairs.tolist()] for pairs in got] == maps.kmap(t_in, t_out, k), (t_in, t_out, k)


# ---------------------------------------------------------------- MinkUNet state_dict

# model/mink_unet.py: (LAYERS, PLANES) of every arch the reference's factory accepts
REFERENCE_ARCHS = {
    "MinkUNet14A": ((1, 1, 1, 1, 1, 1, 1, 1), (32, 64, 128, 256, 128, 128, 96, 96)),
    "MinkUNet14B": ((1, 1, 1, 1, 1, 1, 1, 1), (32, 64, 128, 256, 128, 128, 128, 128)),
    "MinkUNet14C": ((1, 1, 1, 1, 1, 1, 1, 1), (32, 64, 128, 256, 192, 192, 128, 128)),
    "MinkUNet14D": ((1, 1, 1, 1, 1, 1, 1, 1), (32, 64, 128, 256, 384, 384, 384, 384)),
    "MinkUNet18A": ((2, 2, 2, 2, 2, 2, 2, 2), (32, 64, 128, 256, 128, 128, 96, 96)),
    "MinkUNet18B": ((2, 2, 2, 2, 2, 2, 2, 2), (32, 64, 128, 256, 128, 128, 128, 128)),
    "MinkUNet18D": ((2, 2, 2, 2, 2, 2, 2, 2), (32, 64, 128, 256, 384, 384, 384, 384)),
    "MinkUNet34A": ((2, 3, 4, 6, 2, 2, 2, 2), (32, 64, 128, 256, 256, 128, 64, 64)),
    "MinkUNet34B": ((2, 3, 4, 6, 2, 2, 2, 2), (32, 64, 128, 256, 256, 128, 64, 32)),
    "MinkUNet34C": ((2, 3, 4, 6, 2, 2, 2, 2), (32, 64, 128, 256, 256, 128, 96, 96)),
}


def expected_state_dict_shapes(cin, cout, layers, planes):
    """Keys and shapes of the reference module, from MinkUNetBase.network_initialization, ResNetBase._make_layer,
    ME's BasicBlock (conv1, norm1, conv2, norm2, downsample) and ME's layers (kernel (K, in, out) or (in, out) for
    K = 1; MinkowskiBatchNorm's BatchNorm1d as .bn)."""
    sd = {}

    def conv(name, k, i, o):
        sd[f"{name}.kernel"] = (k ** 3, i, o) if k > 1 else (i, o)

    def bn(name, n):
        for leaf in ("weight", "bias", "running_mean", "running_var"):
            sd[f"{name}.bn.{leaf}"] = (n,)
        sd[f"{name}.bn.num_batches_tracked"] = ()

    def layer(name, inplanes, p, n):
        for j in range(n):
            conv(f"{name}.{j}.conv1", 3, inplanes, p)
            bn(f"{name}.{j}.norm1", p)
            conv(f"{name}.{j}.conv2", 3, p, p)
            bn(f"{name}.{j}.norm2", p)
            if j == 0 and inplanes != p:
                conv(f"{name}.{j}.downsample.0", 1, inplanes, p)
                bn(f"{name}.{j}.downsample.1", p)
            inplanes = p
        return p

    conv("conv0p1s1", 5, cin, 32)
    bn("bn0", 32)
    inplanes = 32
    for s, (c, b) in enumerate((("conv1p1s2", "bn1"), ("conv2p2s2", "bn2"), ("conv3p4s2", "bn3"),
                                ("conv4p8s2", "bn4"))):
        conv(c, 2, inplanes, inplanes)
        bn(b, inplanes)
        inplanes = layer(f"block{s + 1}", inplanes, planes[s], layers[s])
    skips = (planes[2], planes[1], planes[0], 32)
    for s, (c, b) in enumerate((("convtr4p16s2", "bntr4"), ("convtr5p8s2", "bntr5"), ("convtr6p4s2", "bntr6"),
                                ("convtr7p2s2", "bntr7"))):
        conv(c, 2, inplanes, planes[4 + s])
        bn(b, planes[4 + s])
        inplanes = layer(f"block{s + 5}", planes[4 + s] + skips[s], planes[4 + s], layers[4 + s])
    conv("final", 1, planes[7], cout)
    return sd


@pytest.mark.parametrize("arch", sorted(REFERENCE_ARCHS))
@pytest.mark.parametrize("cin", [56, 48])
def test_state_dict_keys_and_shapes_equal_the_reference(arch, cin):
    assert set(ARCHS) == set(REFERENCE_ARCHS)
    m = mink_unet(in_channels=cin, out_channels=768, D=3, arch=arch)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == expected_state_dict_shapes(cin, 768, *REFERENCE_ARCHS[arch])


def test_minkunet34a_table():
    sd = mink_unet(56, 768, arch="MinkUNet34A").state_dict()
    table = {"conv0p1s1.kernel": (125, 56, 32), "bn0.bn.running_var": (32,), "block2.0.downsample.0.kernel": (32, 64),
             "convtr4p16s2.kernel": (8, 256, 256), "block5.0.downsample.0.kernel": (384, 256),
             "convtr5p8s2.kernel": (8, 256, 128), "block8.0.conv1.kernel": (27, 96, 64), "final.kernel": (64, 768)}
    for k, shape in table.items():
        assert tuple(sd[k].shape) == shape, k


def test_initialisation_follows_the_reference():
    torch.manual_seed(0)
    m = mink_unet(56, 768, arch="MinkUNet34A")
    k = m.block3[0].conv1.kernel                                             # (27, 64, 128): kaiming fan_out
    assert abs(k.std().item() - (2.0 / (27 * 128)) ** 0.5) < 0.05 * (2.0 / (27 * 128)) ** 0.5
    tr = m.convtr4p16s2.kernel                                               # ME default: U(+-1/sqrt(out * K))
    assert tr.abs().max().item() <= 1 / (256 * 8) ** 0.5
    assert (m.bn0.bn.weight == 1).all() and (m.bn0.bn.bias == 0).all() and m.bn0.bn.momentum == 0.1


# ---------------------------------------------------------------- validation

@pytest.mark.parametrize("kw", [dict(kernel_size=3, stride=2), dict(kernel_size=4), dict(kernel_size=2, stride=1),
                                dict(kernel_size=1, stride=2), dict(kernel_size=3, dilation=2),
                                dict(kernel_size=3, dimension=2), dict(kernel_size=3, bias=True)])
def test_unsupported_convolutions_raise_at_construction(kw):
    with pytest.raises(NotImplementedError):
        sp.Convolution(4, 4, **kw)


@pytest.mark.parametrize("kw", [dict(kernel_size=3, stride=1), dict(kernel_size=2, stride=1),
                                dict(kernel_size=4, stride=4)])
def test_unsupported_transposed_convolutions_raise_at_construction(kw):
    with pytest.raises(NotImplementedError):
        sp.ConvolutionTranspose(4, 4, **kw)


def test_factory_rejects_unknown_arch_and_dimension():
    with pytest.raises(ValueError):
        mink_unet(3, 20, arch="MinkUNet50")
    with pytest.raises(NotImplementedError):
        mink_unet(3, 20, D=2, arch="MinkUNet14A")


def test_sparse_tensor_needs_cuda_fp32_features():
    with pytest.raises(ValueError, match="float32 CUDA"):
        sp.SparseTensor(torch.zeros(4, 3), torch.zeros(4, 4, dtype=torch.int32))
    with pytest.raises(ValueError, match="float32 CUDA"):
        sp.SparseTensor(torch.zeros(4, 3, dtype=torch.float64), torch.zeros(4, 4, dtype=torch.int32))


def _off(*v):
    return (C.c_int64 * len(v))(*v)


@pytest.mark.parametrize("call,msg", [
    (lambda l: l.sgb_coord_map_build(0, 16, 16, 16, None), b"N = 0"),
    (lambda l: l.sgb_coord_map_build(10, None, 16, 16, None), b"null coordinates"),
    (lambda l: l.sgb_coord_map_build(10, 16, None, 16, None), b"null table"),
    (lambda l: l.sgb_coord_map_build(10, 16, 16, None, None), b"null status"),
    (lambda l: l.sgb_coord_map_build(10, 20, 16, 16, None), b"not 16-byte aligned"),
    (lambda l: l.sgb_coord_stride(10, 16, 0, 16, 16, 16, None), b"tensor stride 0"),
    (lambda l: l.sgb_coord_stride(10, 16, 1, 16, None, 16, None), b"out_coords"),
    (lambda l: l.sgb_kernel_map_count(10, 16, 16, 10, 16, 4, 1, 16, 16, None), b"kernel size 4"),
    (lambda l: l.sgb_kernel_map_count(10, 16, None, 10, 16, 3, 1, 16, 16, None), b"null input table"),
    (lambda l: l.sgb_kernel_map_count(10, 16, 16, 10, 16, 3, 1, 16, None, None), b"null offsets"),
    (lambda l: l.sgb_kernel_map_fill(10, 16, 16, 0, 16, 3, 1, 16, 16, None), b"N_out = 0"),
    (lambda l: l.sgb_kernel_map_fill(10, 16, 16, 10, 16, 3, 1, 16, None, None), b"pairs"),
    (lambda l: l.sgb_sparse_conv_forward(0, _off(0), 16, 0, 4, 3, 16, 16, 4, 3, 16, None), b"K = 0"),
    (lambda l: l.sgb_sparse_conv_forward(126, _off(*[0] * 127), 16, 0, 4, 3, 16, 16, 4, 3, 16, None), b"K = 126"),
    (lambda l: l.sgb_sparse_conv_forward(1, _off(0, 2), 16, 0, 4, 0, 16, 16, 4, 3, 16, None), b"C_in = 0"),
    (lambda l: l.sgb_sparse_conv_forward(1, _off(0, 2), 16, 0, 4, 3, 16, 16, 4, -1, 16, None), b"C_out = -1"),
    (lambda l: l.sgb_sparse_conv_forward(1, None, 16, 0, 4, 3, 16, 16, 4, 3, 16, None), b"null offsets"),
    (lambda l: l.sgb_sparse_conv_forward(2, _off(0, 3, 2), 16, 0, 4, 3, 16, 16, 4, 3, 16, None), b"decrease"),
    (lambda l: l.sgb_sparse_conv_forward(1, _off(0, 2), None, 0, 4, 3, 16, 16, 4, 3, 16, None), b"pairs"),
    (lambda l: l.sgb_sparse_conv_forward(1, _off(0, 2), 16, 0, 4, 3, None, 16, 4, 3, 16, None), b"null x"),
    (lambda l: l.sgb_sparse_conv_backward_input(1, _off(0, 2), 16, 0, 4, 3, None, 16, 4, 3, 16, None), b"null dx"),
    (lambda l: l.sgb_sparse_conv_backward_weight(1, _off(0, 2), 16, 0, 4, 3, 16, 4, 3, 16, None, 16, None),
     b"workspace"),
    (lambda l: l.sgb_sparse_conv_backward_weight(200, _off(0, 2), 16, 0, 4, 3, 16, 4, 3, 16, 16, 16, None),
     b"K = 200"),
])
def test_entry_points_validate_before_cuda(call, msg):
    lib = _lib.load()
    assert call(lib) == -1
    assert msg in lib.sgb_last_error()


def test_workspace_queries_reject_what_the_calls_reject():
    lib = _lib.load()
    assert lib.sgb_coord_map_bytes(0) == 0 and lib.sgb_coord_map_bytes(100) >= 4 * 200
    assert lib.sgb_coord_stride_workspace_bytes(-1) == 0
    assert lib.sgb_kernel_map_workspace_bytes(0, 3) == 0
    assert lib.sgb_sparse_conv_backward_weight_workspace_bytes(0, _off(0), 3, 3) == 0
    assert lib.sgb_sparse_conv_backward_weight_workspace_bytes(1, _off(0, 5), 0, 3) == 0
