"""The half-precision sparse convolution (fp16 / bf16 features, tensor cores) against the float64 restatement of
tests/sparse_ref.py.  x, the kernel and dy are rounded to the half type first and the restatement is computed from those
rounded values, so what is left is the kernels' own arithmetic: fp32 accumulation (half x half products are exact in
fp32) and, for out and dx, the one final rounding to the half type.  With S the same product of absolute values and u
the unit roundoff (2^-8 bf16, 2^-11 fp16):

    out, dx    |got - ref| <= 1e-5 S + u (|ref| + 1e-5 S)   (+ 2^-25 for fp16, half its subnormal spacing)
    dW (fp32)  |got - ref| <= 1e-5 S                        (the fp32 products' own bound)

u (|ref| + 1e-5 S) is the rounding of the accumulated value, which lies within 1e-5 S of ref.  Also: every layer
product at the sizes distillation trains on, under bf16 autocast; bitwise reproducibility; dtype routing of every
layer; and short fp16 / bf16 training loops.  Run with -s for the worst err / bound ratios."""
import pytest
import torch

import sparse_ref as ref
from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200 import sparse as sp
from semantic_gaussians_b200.mink_unet import mink_unet
from semantic_gaussians_b200.scene_synth import surface_voxels
from semantic_gaussians_b200.voxelize import distill_targets
from test_sparse_gpu import DEV, _layer_case, _room_input

pytestmark = pytest.mark.gpu

HALF = {"fp16": torch.float16, "bf16": torch.bfloat16}
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


def _within(got, want, S, rounding_u, floor, what):
    """|got - want| <= 1e-5 S + u (|want| + 1e-5 S) + floor everywhere; returns the worst err / bound.  For out and
    dx the rounding term dominates the bound, so their ratio reads close to 1 whenever an element rounds by nearly
    half a unit; for dW (u = 0) it is the accumulation error over 1e-5 S."""
    err = (got.to(want.device, torch.float64) - want).abs()
    acc = 1e-5 * S
    bound = acc + rounding_u * (want.abs() + acc) + floor
    ok = err <= bound + 1e-30
    worst = (err / bound.clamp_min(1e-30)).max().item()
    assert bool(ok.all()), f"{what}: worst err {err.max().item():.3g}, worst err / bound {worst:.3g}"
    return worst


def check_half_products(x, W, dy, km, rk, transposed, n_out):
    """One layer forward and backward through the half path (x, dy in the half type, W the fp32 parameter), against
    the float64 restatement over the pairs rk on the rounded values.  Returns (out, dx, dW) and the worst
    err / bound ratio of each."""
    dt = x.dtype
    u, floor = UNIT[dt], (2.0 ** -25 if dt == torch.float16 else 0.0)
    xg, Wg = x.detach().clone().requires_grad_(True), W.detach().float().clone().requires_grad_(True)
    out = sp._HalfSparseConvFunction.apply(xg, Wg, km, transposed, n_out)
    assert out.dtype == dt
    out.backward(dy)
    assert xg.grad.dtype == dt and Wg.grad.dtype == torch.float32
    x64, W64, dy64 = x.detach().double(), W.detach().to(dt).double(), dy.double()
    n_in = x.shape[0]
    ratios = {"out": _within(out.detach(), ref.conv(x64, W64, rk, n_out, transposed),
                             ref.conv(x64.abs(), W64.abs(), rk, n_out, transposed), u, floor, "forward")}
    Wt = W64.transpose(1, 2)
    ratios["dx"] = _within(xg.grad, ref.conv(dy64, Wt, rk, n_in, not transposed),
                           ref.conv(dy64.abs(), Wt.abs(), rk, n_in, not transposed), u, floor, "dx")
    dW, bW = torch.zeros_like(W64), torch.zeros_like(W64)
    for d, pairs in enumerate(rk):
        if len(pairs):
            p = torch.as_tensor(pairs, dtype=torch.int64, device=x.device)
            xs, ys = (p[:, 1], p[:, 0]) if transposed else (p[:, 0], p[:, 1])
            dW[d] = x64[xs].T @ dy64[ys]
            bW[d] = x64[xs].abs().T @ dy64[ys].abs()
    ratios["dW"] = _within(Wg.grad, dW, bW, 0.0, 0.0, "dW")
    return (out.detach(), xg.grad, Wg.grad), ratios


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("cin", [1, 3, 32, 56, 96, 384])
@pytest.mark.parametrize("cout", [1, 32, 64, 256])
@pytest.mark.parametrize("k,stride,transposed", [(3, 1, False), (5, 1, False), (2, 2, False), (2, 2, True)])
def test_half_products_match_float64(cin, cout, k, stride, transposed, dtype):
    dt = HALF[dtype]
    km, rk, n_in, n_out = _layer_case(k, stride, transposed)
    g = torch.Generator().manual_seed(cin * 1000 + cout)
    x = torch.randn(n_in, cin, generator=g, dtype=torch.float64)
    W = torch.randn(km.K, cin, cout, generator=g, dtype=torch.float64) / cin ** 0.5
    dy = torch.randn(n_out, cout, generator=g, dtype=torch.float64)
    check_half_products(x.to(dt).to(DEV), W.float().to(DEV), dy.to(dt).to(DEV), km, rk, transposed, n_out)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("cin,cout", [(65, 130), (130, 65), (8, 3)])
def test_half_products_of_widths_off_the_fast_path(cin, cout, dtype):
    """Widths that are not a multiple of 8 elements in x, dy or the kernel: the staging path on one side or both."""
    dt = HALF[dtype]
    for k, stride, transposed in [(3, 1, False), (2, 2, True)]:
        km, rk, n_in, n_out = _layer_case(k, stride, transposed)
        g = torch.Generator().manual_seed(cin + 7 * cout)
        x = torch.randn(n_in, cin, generator=g).to(dt).to(DEV)
        W = (torch.randn(km.K, cin, cout, generator=g) / cin ** 0.5).to(DEV)
        dy = torch.randn(n_out, cout, generator=g).to(dt).to(DEV)
        check_half_products(x, W, dy, km, rk, transposed, n_out)


# the weight-gradient chunk cases of test_sparse_scale_gpu.py: 1, 1, 2, 2 and 4 chunks of 2048 pairs at the centre
# offset, partial inner blocks and steps, and several chunks per offset of the transposed k = 2 layer at 50 k rows
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("cin,cout", [(56, 32), (96, 96), (65, 130)])
@pytest.mark.parametrize("k,N", [(3, 2047), (3, 2048), (3, 2049), (3, 2048 + 129), (3, 3 * 2048 + 17), (2, 50_000)])
def test_half_weight_gradient_chunk_boundaries(k, N, cin, cout, dtype):
    dt = HALF[dtype]
    rows = ref.random_rows("box", N, 1, seed=N)
    transposed = k == 2
    km, rk, n_in, n_out = _layer_case(k, 2 if transposed else 1, transposed, rows)
    if transposed:
        assert min(km.counts) > 2 * 2048
    else:
        assert km.counts[13] == N
    g = torch.Generator(device=DEV).manual_seed(N + cin)
    x = torch.randn(n_in, cin, device=DEV, generator=g).to(dt)
    W = torch.randn(km.K, cin, cout, device=DEV, generator=g) / cin ** 0.5
    dy = torch.randn(n_out, cout, device=DEV, generator=g).to(dt)
    _, ratios = check_half_products(x, W, dy, km, rk, transposed, n_out)
    print(f"\n  {dtype} k={k} N={N} {cin}->{cout}: " + ", ".join(f"{p} {r:.2e}" for p, r in ratios.items()))


def _offset_pairs(km):
    return [km.pairs[a:b] for a, b in zip(km.offsets_host[:km.K], km.offsets_host[1:km.K + 1])]


@pytest.mark.parametrize("kind", ["room_20k", "surface_600k"])
def test_bf16_network_layer_products_match_float64(kind, monkeypatch):
    """Every sparse convolution of MinkUNet34A in train mode under bf16 autocast, re-checked on the bf16 input, the
    rounded kernel and the bf16 upstream gradient the network gave it."""
    torch.manual_seed(0)
    if kind == "room_20k":
        locs, feats, _ = _room_input()
    else:
        locs, feats = surface_voxels(1_000_000, DEV)
        assert 500_000 < locs.shape[0] < 700_000
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    model = mink_unet(56, 768, arch="MinkUNet34A").to(DEV)
    params = dict(model.named_parameters())
    names = {id(m.kernel): n for n, m in model.named_modules() if isinstance(m, (sp.Convolution,
                                                                                 sp.ConvolutionTranspose))}
    calls = []
    apply = sp._HalfSparseConvFunction.apply

    def capture(x, kernel, kmap, transposed, n_out):
        out = apply(x, kernel, kmap, transposed, n_out)
        rec = dict(name=names[id(kernel)], x=x.detach(), W=kernel.detach(), km=kmap, transposed=transposed,
                   n_out=n_out, out=out.detach())
        out.register_hook(lambda g: rec.__setitem__("dy", g))
        calls.append(rec)
        return out

    with monkeypatch.context() as m:
        m.setattr(sp._HalfSparseConvFunction, "apply", capture)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(sp.SparseTensor(feats, locs))
        assert out.F.dtype == torch.bfloat16
        out.F.backward(torch.randn(out.F.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1)))
    del out
    assert len(calls) == sum(1 for n, p in params.items() if n.endswith(".kernel") and p.dim() == 3)
    print(f"\n  {kind}: {locs.shape[0]} voxels, network peak {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.2f} GiB;"
          " worst err / bound per layer")
    worst = {"out": (0.0, ""), "dx": (0.0, ""), "dW": (0.0, "")}
    while calls:
        c = calls.pop(0)
        km = c["km"]
        assert c["x"].dtype == c["dy"].dtype == torch.bfloat16, c["name"]
        (o, _, dW), ratios = check_half_products(c["x"], c["W"], c["dy"], km, _offset_pairs(km), c["transposed"],
                                                 c["n_out"])
        assert torch.equal(o, c["out"]), c["name"]
        grad = params[c["name"] + ".kernel"].grad
        assert grad.dtype == torch.float32 and torch.equal(dW, grad), c["name"]
        K, cin, cout = c["W"].shape
        print(f"  {c['name']:<22} k^3={K:<3} {cin:>3} -> {cout:<3} pairs {km.offsets_host[K]:>9}  "
              f"out {ratios['out']:.2e}  dx {ratios['dx']:.2e}  dW {ratios['dW']:.2e}")
        for p, r in ratios.items():
            worst[p] = max(worst[p], (r, c["name"]))
        del c, o, dW
    print("  worst: " + ", ".join(f"{p} {r:.2e} ({n})" for p, (r, n) in worst.items()))


def test_two_bf16_passes_are_bitwise_equal_at_600k():
    torch.manual_seed(0)
    locs, feats = surface_voxels(1_000_000, DEV)
    model = mink_unet(56, 96, arch="MinkUNet34A").to(DEV)
    dy = torch.randn(locs.shape[0], 96, device=DEV).bfloat16()
    results = []
    for _ in range(2):
        model.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(sp.SparseTensor(feats, locs))
        out.F.backward(dy)
        results.append((out.F.detach().clone(), [p.grad.clone() for p in model.parameters()]))
        del out
    assert results[0][0].dtype == torch.bfloat16 and torch.equal(results[0][0], results[1][0])
    for a, b in zip(results[0][1], results[1][1]):
        assert a.dtype == torch.float32 and torch.equal(a, b)


# ---------------------------------------------------------------- routing

class _Spy:
    """_lib.load() stand-in that records the name of every native entry point sparse.py takes from it."""

    def __init__(self, lib):
        self.lib, self.names = lib, []

    def __getattr__(self, name):
        self.names.append(name)
        return getattr(self.lib, name)


def _run(model, feats, locs, autocast_dtype, monkeypatch):
    """One forward + backward; returns the entry points called and the dtype of the features every layer gave and
    (but for the first, which takes the network's input) was given: the outputs of cat and the residual + are inputs
    of later layers."""
    spy = _Spy(_lib.load())
    dtypes = {}
    mods = {m: n for n, m in model.named_modules() if isinstance(m, (sp.Convolution, sp.ConvolutionTranspose,
                                                                      sp.BatchNorm, sp.ReLU))}

    def hook(mod, inp, out):
        dtypes[mods[mod]] = out.F.dtype
        if mods[mod] != "conv0p1s1":
            dtypes[mods[mod] + " input"] = inp[0].F.dtype

    hooks = [m.register_forward_hook(hook) for m in mods]
    try:
        with monkeypatch.context() as mp:
            mp.setattr(_lib, "load", lambda: spy)
            with torch.autocast("cuda", dtype=autocast_dtype or torch.bfloat16, enabled=autocast_dtype is not None):
                out = model(sp.SparseTensor(feats, locs))
            out.F.float().sum().backward()
    finally:
        for h in hooks:
            h.remove()
    return set(n for n in spy.names if n.startswith("sgb_sparse_conv")), dtypes, out.F.dtype


FP32_CALLS = {"sgb_sparse_conv_forward", "sgb_sparse_conv_backward_input", "sgb_sparse_conv_backward_weight",
              "sgb_sparse_conv_backward_weight_workspace_bytes"}


@pytest.mark.parametrize("dtype,autocast", [("bf16", True), ("fp16", True), ("bf16", False), ("fp16", False)])
def test_half_features_take_the_half_path_in_every_layer(dtype, autocast, monkeypatch):
    """Under autocast, fp32 features give half outputs from every sparse layer, BatchNorm, ReLU, cat and the residual
    +; explicit half features do the same without autocast.  Only the half entry points are called."""
    dt = HALF[dtype]
    torch.manual_seed(0)
    locs, feats, _ = _room_input(8_000)
    model = mink_unet(56, 64, arch="MinkUNet34A").to(DEV)
    feats = feats if autocast else feats.to(dt)
    called, dtypes, out_dtype = _run(model, feats, locs, dt if autocast else None, monkeypatch)
    assert called and not called & FP32_CALLS, called
    assert {"sgb_sparse_conv_half_forward", "sgb_sparse_conv_half_backward_input",
            "sgb_sparse_conv_half_backward_weight"} <= called
    assert out_dtype == dt and set(dtypes.values()) == {dt}, dtypes
    assert all(p.grad is not None and p.grad.dtype == torch.float32 for p in model.parameters())


def test_fp32_features_outside_autocast_call_the_fp32_entry_points(monkeypatch):
    torch.manual_seed(0)
    locs, feats, _ = _room_input(8_000)
    model = mink_unet(56, 64, arch="MinkUNet14A").to(DEV)
    called, dtypes, out_dtype = _run(model, feats, locs, None, monkeypatch)
    assert called == FP32_CALLS, called
    assert out_dtype == torch.float32 and set(dtypes.values()) == {torch.float32}


# ---------------------------------------------------------------- training

@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_half_distill_loop_lowers_the_loss(dtype):
    """test_sparse_gpu.py's distill loop under autocast: bf16 as it is, fp16 through torch.amp.GradScaler."""
    dt = HALF[dtype]
    torch.manual_seed(0)
    locs, feats, vox_ind = _room_input(8_000)
    P = int(vox_ind.max().item()) + 1
    mask_full = (torch.rand(P, device=DEV) < 0.6)
    gen = torch.Generator(device=DEV).manual_seed(2)
    feat = torch.nn.functional.normalize(torch.randn(int(mask_full.sum()), 64, device=DEV, generator=gen), dim=-1)
    mask, features_gt = distill_targets(vox_ind, mask_full, feat)
    model = mink_unet(56, 64, arch="MinkUNet14A").to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", enabled=dt == torch.float16)
    losses = []
    for _ in range(5):
        locs_aug = locs.clone()
        locs_aug[:, 1:4] += (torch.rand(3) * 100).int().to(DEV)
        with torch.autocast("cuda", dtype=dt):
            output = model(sp.SparseTensor(feats, locs_aug)).F[mask]
            assert output.dtype == dt
            norm_mask = features_gt.norm(dim=-1) > 0
            loss = (1 - torch.nn.CosineSimilarity()(output[norm_mask].float(), features_gt[norm_mask])).mean()
        opt.zero_grad()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        losses.append(loss.item())
    assert all(p.dtype == torch.float32 for p in model.parameters())
    assert losses[-1] < losses[0], losses
