"""The sparse convolution at the sizes distillation trains on (0.6 - 1 M voxels), against the restatement of
tests/sparse_ref.py on the kernels' own inputs, so that what is measured is the kernels' own arithmetic:

* coordinate maps of strides 1 - 16 and every kernel map MinkUNet builds, bit for bit with the sorting restatement
  (TensorMaps), on the `room` scene at 1 M Gaussians, four copies of one surface cloud that differ only in b, and
  ~1 M "low_bits" rows;
* every sparse convolution of a MinkUNet34A forward + backward in train mode, re-run on the input, kernel and upstream
  gradient captured from the network: out, dx and dW within 1e-5 of the same product of absolute values in float64,
  dW bitwise equal to the network's kernel gradient;
* weight gradients whose offsets are cut into 1, 2 and 4 chunks of the chunked reduction, with partial tiles.

Run with -s for the worst err / bound ratio of each layer and product and the peak device memory of each test."""
import numpy as np
import pytest
import torch

import sparse_ref as ref
from semantic_gaussians_b200 import sparse as sp
from semantic_gaussians_b200.mink_unet import mink_unet
from semantic_gaussians_b200.scene_synth import surface_voxels
from test_sparse_gpu import DEV, _layer_case, _room_input, check_products

pytestmark = pytest.mark.gpu

K_CHUNK = 2048      # pairs per weight-gradient partial in sparse_conv.cu


@pytest.fixture(autouse=True)
def _peak_memory():
    torch.cuda.init()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    print(f"\n  peak memory allocated: {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.2f} GiB")


def _cloud(kind):
    if kind == "room_1m":
        rows = _room_input(1_000_000)[0]
        assert 900_000 < rows.shape[0] < 1_100_000
    elif kind == "surface_copies":   # rows equal in x, y, z appear once per batch
        one = surface_voxels(300_000, DEV)[0]
        assert 150_000 < one.shape[0] < 350_000
        rows = torch.cat([torch.cat([torch.full_like(one[:, :1], b), one[:, 1:]], 1) for b in range(4)])
    else:
        rows = torch.from_numpy(ref.random_rows("low_bits", 1_000_000, 1, seed=1)).to(DEV)
    return rows


@pytest.mark.parametrize("kind", ["room_1m", "surface_copies", "low_bits_1m"])
def test_maps_at_scale_equal_the_restatement(kind):
    rows = _cloud(kind)
    mgr = sp.CoordinateManager(rows)
    maps = ref.TensorMaps(rows)
    for t in (1, 2, 4, 8, 16):
        assert torch.equal(mgr.map(t).coords, maps.at(t)), t
    print(f"\n  {kind}: rows by stride {[mgr.map(t).n for t in (1, 2, 4, 8, 16)]}")
    for key in ref.MINKUNET_KMAPS:
        km, want = mgr.kernel_map(*key), maps.kmap(*key)
        assert list(km.offsets_host) == [0] + np.cumsum([len(p) for p in want]).tolist(), key
        assert torch.equal(km.pairs.long(), torch.cat(want)), key
        del mgr.kernel_maps[key], maps.kmaps[key]


def _offset_pairs(km):
    return [km.pairs[a:b] for a, b in zip(km.offsets_host[:km.K], km.offsets_host[1:km.K + 1])]


@pytest.mark.parametrize("kind", ["room_20k", "surface_600k"])
def test_network_layer_products_match_float64(kind, monkeypatch):
    """Every sparse convolution of MinkUNet34A in train mode, on the tensors the network gave it.  These include the
    layers whose gradients sit behind the network test's relaxed bound (conv0p1s1, block7.0.conv1)."""
    torch.manual_seed(0)
    if kind == "room_20k":
        locs, feats, _ = _room_input()
    else:
        locs, feats = surface_voxels(1_000_000, DEV)
        assert 500_000 < locs.shape[0] < 700_000
    model = mink_unet(56, 768, arch="MinkUNet34A").to(DEV)
    params = dict(model.named_parameters())
    names = {id(m.kernel): n for n, m in model.named_modules() if isinstance(m, (sp.Convolution,
                                                                                 sp.ConvolutionTranspose))}
    calls = []
    apply = sp._SparseConvFunction.apply

    def capture(x, kernel, kmap, transposed, n_out):
        out = apply(x, kernel, kmap, transposed, n_out)
        rec = dict(name=names[id(kernel)], x=x.detach(), W=kernel.detach(), km=kmap, transposed=transposed,
                   n_out=n_out, out=out.detach())
        out.register_hook(lambda g: rec.__setitem__("dy", g))
        calls.append(rec)
        return out

    with monkeypatch.context() as m:
        m.setattr(sp._SparseConvFunction, "apply", capture)
        out = model(sp.SparseTensor(feats, locs))
        out.F.backward(torch.randn(out.F.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1)))
    del out
    assert len(calls) == sum(1 for n, p in params.items() if n.endswith(".kernel") and p.dim() == 3)
    print(f"\n  {kind}: {locs.shape[0]} voxels; worst err / sum of |products| per layer (tolerance 1e-5)")
    worst = {"out": (0.0, ""), "dx": (0.0, ""), "dW": (0.0, "")}
    while calls:
        c = calls.pop(0)
        km = c["km"]
        (o, _, dW), ratios = check_products(c["x"], c["W"], c["dy"], km, _offset_pairs(km), c["transposed"],
                                            c["n_out"])
        assert torch.equal(o, c["out"]), c["name"]
        assert torch.equal(dW, params[c["name"] + ".kernel"].grad), c["name"]
        K, cin, cout = c["W"].shape
        print(f"  {c['name']:<22} k^3={K:<3} {cin:>3} -> {cout:<3} pairs {km.offsets_host[K]:>9} max/offset "
              f"{max(km.counts):>8}  out {ratios['out']:.2e}  dx {ratios['dx']:.2e}  dW {ratios['dW']:.2e}")
        for p, r in ratios.items():
            worst[p] = max(worst[p], (r, c["name"]))
        del c, o, dW
    print("  worst: " + ", ".join(f"{p} {r:.2e} ({n})" for p, (r, n) in worst.items()))


def test_two_passes_are_bitwise_equal_at_600k():
    torch.manual_seed(0)
    locs, feats = surface_voxels(1_000_000, DEV)
    model = mink_unet(56, 96, arch="MinkUNet34A").to(DEV)
    dy = torch.randn(locs.shape[0], 96, device=DEV)
    results = []
    for _ in range(2):
        model.zero_grad()
        out = model(sp.SparseTensor(feats, locs))
        out.F.backward(dy)
        results.append((out.F.detach().clone(), [p.grad.clone() for p in model.parameters()]))
        del out
    assert torch.equal(results[0][0], results[1][0])
    for a, b in zip(results[0][1], results[1][1]):
        assert torch.equal(a, b)


# The centre offset of a stride-1 k = 3 layer pairs every row with itself: N rows give it exactly N pairs, so N picks
# the chunk boundaries (1, 1, 2, 2 and 4 chunks), partial 128-pair inner blocks and partial 16-pair steps.  The
# transposed k = 2 layer at 50 k rows has ~N / 8 pairs per offset, several chunks each.
@pytest.mark.parametrize("cin,cout", [(56, 32), (96, 96), (65, 130)])
@pytest.mark.parametrize("k,N", [(3, 2047), (3, 2048), (3, 2049), (3, 2048 + 129), (3, 3 * 2048 + 17), (2, 50_000)])
def test_weight_gradient_chunk_boundaries(k, N, cin, cout):
    rows = ref.random_rows("box", N, 1, seed=N)
    transposed = k == 2
    km, rk, n_in, n_out = _layer_case(k, 2 if transposed else 1, transposed, rows)
    if transposed:
        assert min(km.counts) > 2 * K_CHUNK
    else:
        assert km.counts[13] == N
    g = torch.Generator(device=DEV).manual_seed(N + cin)
    x = torch.randn(n_in, cin, device=DEV, generator=g)
    W = torch.randn(km.K, cin, cout, device=DEV, generator=g) / cin ** 0.5
    dy = torch.randn(n_out, cout, device=DEV, generator=g)
    _, ratios = check_products(x, W, dy, km, rk, transposed, n_out)
    print(f"\n  k={k} N={N} {cin}->{cout}: " + ", ".join(f"{p} {r:.2e}" for p, r in ratios.items()))
