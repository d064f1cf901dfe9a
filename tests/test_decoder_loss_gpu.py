"""Decoded feature-map loss (semantic.decoded_feature_map_loss_and_grads, sgb_decoded_feature_loss) on the GPU: loss,
pixel count and the three gradients against float64 torch autograd of x = W r + b followed by the reference's
expressions (distill.py:111-124) at every compact width, decoded width, target dtype and image shape its kernels
branch on; the identity decoder against feature_map_loss_and_grad; edge cases; synchronisation, reproducibility and
memory at K4's view size; and a short fit of a compact field plus decoder through render_chn."""
import pytest
import torch
from feature_loss_ref import feature_loss

from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200.semantic import decoded_feature_map_loss_and_grads, feature_map_loss_and_grad

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LOSS_TYPES = ("cosine", "l1", "l2")


def _inputs(c, C, H, W, dtype, bias, seed):
    """render / decoder / target with: target pixels that are all zero, target pixels with a single non-zero (last)
    channel, and render pixels that are zero (a decoded pixel of exactly zero without a bias).  r, W and b are
    multiples of 1/16, 1/64 and 1/1024 small enough that x = W r + b is exact in fp32 in any order of summation: the
    sign of x - y (l1) is then the same for the kernel and the float64 reference, and ties x = y give sign(0) in both."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = torch.randn((c, H, W), generator=g, device=DEV) * torch.rand((1, H, W), generator=g, device=DEV).add_(0.1)
    r = (r * 16).round_().clamp_(-127, 127) / 16
    w = ((torch.randn((C, c), generator=g, device=DEV) / c ** 0.5 * 64).round_().clamp_(-255, 255) / 64)
    b = (0.3 * torch.randn(C, generator=g, device=DEV) * 1024).round_() / 1024 if bias else None
    u = torch.rand((H, W), generator=g, device=DEV)
    r[:, u < 0.05] = 0
    r[:, 0, 0] = 0
    x = torch.einsum("kc,chw->khw", w.double(), r.double())
    if b is not None:
        x += b.double()[:, None, None]
    y = (0.6 * x.float() + torch.randn((C, H, W), generator=g, device=DEV)).to(dtype)
    y[:, (u >= 0.05) & (u < 0.15)] = 0
    if C > 1:
        y[:-1, (u >= 0.15) & (u < 0.2)] = 0
    return r.contiguous(), w, b, y.contiguous()


def _reference(r, w, b, y, loss_type):
    """float64: (loss, dL/dr, dL/dW, dL/db, pixels averaged over, decoded x), feature_loss_ref.feature_loss with one
    row per pixel of x = W r + b, and its gradient taken back through the decoder by autograd."""
    C = w.shape[0]
    _, H, W = r.shape
    rl = r.double().requires_grad_(True)
    wl = w.double().requires_grad_(True)
    bl = b.double().requires_grad_(True) if b is not None else None
    xi = torch.einsum("kc,chw->khw", wl, rl)
    if bl is not None:
        xi = xi + bl[:, None, None]
    loss, n, g = feature_loss(xi.permute(1, 2, 0).reshape(-1, C), y.permute(1, 2, 0).reshape(-1, C), loss_type)
    xi.backward(g.reshape(H, W, C).permute(2, 0, 1))
    return loss, rl.grad, wl.grad, bl.grad if bl is not None else None, n, xi.detach()


def _abi(r, w, b, y, loss_type):
    """The C entry point directly: (loss[2] on the host, dL/dr, dL/dW, dL/db)."""
    C, c = w.shape
    N = r.shape[1] * r.shape[2]
    lib = _lib.load()
    out = torch.empty(2, dtype=torch.float64, device=DEV)
    gr, gw = torch.empty_like(r), torch.empty_like(w)
    gb = torch.empty_like(b) if b is not None else None
    ws = torch.empty(lib.sgb_decoded_feature_loss_workspace_bytes(C, c, N), dtype=torch.uint8, device=DEV)
    dtype = _lib.FEAT_F16 if y.dtype == torch.float16 else _lib.FEAT_F32
    lt = {"cosine": _lib.FEATLOSS_COSINE, "l1": _lib.FEATLOSS_L1, "l2": _lib.FEATLOSS_L2}[loss_type]
    _lib.check(lib.sgb_decoded_feature_loss(C, c, N, r.data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None,
                                            y.data_ptr(), dtype, lt, gr.data_ptr(), gw.data_ptr(),
                                            gb.data_ptr() if gb is not None else None, ws.data_ptr(), out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
    return out.cpu(), gr, gw, gb


def _check(r, w, b, y, loss_type):
    loss, gr, gw, gb = decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=loss_type)
    want_loss, want_r, want_w, want_b, want_n, x = _reference(r, w, b, y, loss_type)
    assert loss.dtype == torch.float64 and loss.ndim == 0 and loss.is_cuda
    assert gr.dtype == torch.float32 and gr.shape == r.shape and gw.shape == w.shape
    assert (gb is None) == (b is None)
    assert abs(float(loss) - want_loss) <= 1e-5 * abs(want_loss) + 1e-7, (float(loss), want_loss)
    # Scales.  For cosine, g_p is the difference of two terms, each at most t_p = 1 / (Nv max(|x_p|, 1e-8)); they
    # cancel where x_p is parallel to y_p (everywhere at C = 1), so each gradient is held to its own largest magnitude
    # or to the size of those terms taken through the contraction, whichever is larger.  Decoded pixels with a clamped
    # norm have a 1e8-times larger g_p: the rest of dL/dR must also match on the scale of the unclamped pixels alone.
    xn = x.norm(dim=0)
    normal = xn >= 1e-8
    t = torch.zeros_like(xn)
    if loss_type == "cosine" and want_n:
        valid = y.double().norm(dim=0) > 0
        t = torch.where(valid, 1.0 / (want_n * xn.clamp_min(1e-8)), t)
    wn = float(w.double().norm(dim=0).max())
    err = (gr.double() - want_r).abs()
    scale = max(float(want_r.abs().max()), wn * float(t.max()))
    assert float(err.max()) <= 1e-5 * scale, (float(err.max()), scale)
    if bool(normal.any()):
        scale_n = max(float(want_r[:, normal].abs().max()), wn * float(t[normal].max()))
        assert float(err[:, normal].max()) <= 1e-5 * scale_n, (float(err[:, normal].max()), scale_n)
    t_w = float((t[None] * r.double().abs()).sum(dim=(1, 2)).max())
    for got, want, t_scale in ((gw, want_w, t_w), (gb, want_b, float(t.sum()))):
        if want is None:
            continue
        e = float((got.double() - want).abs().max())
        s = max(float(want.abs().max()), t_scale)
        assert e <= 1e-4 * s, (e, s)
    assert _abi(r, w, b, y, loss_type)[0][1].item() == want_n


# (c, C, H, W): c pads to 16 / 32 / 64 / 128 columns; C is walked in chunks of 64 rows (5, 768 and 1 leave a partial
# chunk); N % 4 == 0 with aligned planes takes the vector loads and stores, the others plain ones; N % 128 != 0 leaves
# a partial pixel block, and N < 128 * 132 runs fewer CTAs than SMs.
SHAPES = [
    (1, 1, 37, 25), (3, 5, 333, 211), (16, 5, 40, 48), (16, 512, 37, 25), (64, 512, 333, 211), (64, 512, 64, 96),
    (128, 768, 37, 25), (128, 768, 48, 64), (3, 1024, 19, 21), (128, 1024, 16, 40), (64, 1, 61, 33), (1, 768, 24, 40),
]


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("c,C,H,W", SHAPES)
def test_matches_float64_torch(c, C, H, W, dtype, bias, loss_type):
    r, w, b, y = _inputs(c, C, H, W, dtype, bias, seed=c * 7 + C + H)
    _check(r, w, b, y, loss_type)


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
def test_misaligned_views(loss_type):
    """Planes that start at an odd element offset (views into larger buffers, after .contiguous() a no-op) take the
    plain-load path and give the same results as aligned copies."""
    r, w, b, y = _inputs(16, 96, 40, 48, torch.float16, True, seed=11)
    rb = torch.empty(r.numel() + 1, device=DEV)
    yb = torch.empty(y.numel() + 1, dtype=y.dtype, device=DEV)
    rb[1:] = r.reshape(-1)
    yb[1:] = y.reshape(-1)
    rv, yv = rb[1:].view(r.shape), yb[1:].view(y.shape)
    assert rv.data_ptr() % 16 and yv.data_ptr() % 8
    got = decoded_feature_map_loss_and_grads(rv, w, yv, bias=b, loss_type=loss_type)
    want = decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=loss_type)
    assert float(got[0]) == float(want[0])
    for g0, g1 in zip(got[1:], want[1:]):
        assert torch.equal(g0, g1)


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("c,H,W", [(5, 37, 25), (64, 64, 96), (128, 333, 211)])
def test_identity_decoder_equals_the_undecoded_loss(c, H, W, dtype, loss_type):
    r, _, _, y = _inputs(c, c, H, W, dtype, False, seed=c + H)
    w = torch.eye(c, device=DEV)
    b = torch.zeros(c, device=DEV)
    loss, gr, _, _ = decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=loss_type)
    want_loss, want_g = feature_map_loss_and_grad(r, y, loss_type)
    assert abs(float(loss) - float(want_loss)) <= 1e-6 * abs(float(want_loss)), (float(loss), float(want_loss))
    assert float((gr - want_g).abs().max()) <= 1e-6 * float(want_g.abs().max())


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
def test_all_zero_target_gives_zero_loss_count_and_gradients(dtype, bias):
    r, w, b, _ = _inputs(16, 300, 48, 64, dtype, bias, seed=1)
    y = torch.zeros((300, 48, 64), dtype=dtype, device=DEV)
    loss, gr, gw, gb = decoded_feature_map_loss_and_grads(r, w, y, bias=b)
    assert float(loss) == 0.0 and not bool(gr.any()) and not bool(gw.any())
    assert gb is None or not bool(gb.any())
    assert _abi(r, w, b, y, "cosine")[0].tolist() == [0.0, 0.0]


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
def test_empty_image(loss_type):
    w = torch.randn(32, 8, device=DEV)
    b = torch.randn(32, device=DEV)
    loss, gr, gw, gb = decoded_feature_map_loss_and_grads(torch.zeros((8, 0, 5), device=DEV), w,
                                                          torch.zeros((32, 0, 5), device=DEV).half(), bias=b,
                                                          loss_type=loss_type)
    assert float(loss) == 0.0 and gr.shape == (8, 0, 5)
    assert not bool(gw.any()) and not bool(gb.any())


def test_parameters_and_non_contiguous_inputs():
    r, w, b, y = _inputs(16, 64, 40, 24, torch.float16, True, seed=2)
    lin = torch.nn.Linear(16, 64, device=DEV)
    with torch.no_grad():
        lin.weight.copy_(w)
        lin.bias.copy_(b)
    for lt in LOSS_TYPES:
        l0, *g0 = decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=lt)
        rt, yt = r.transpose(1, 2).contiguous().transpose(1, 2), y.transpose(1, 2).contiguous().transpose(1, 2)
        assert not rt.is_contiguous() and not yt.is_contiguous()
        l1, *g1 = decoded_feature_map_loss_and_grads(rt, lin.weight, yt, bias=lin.bias, loss_type=lt)
        assert float(l0) == float(l1) and all(torch.equal(a, b_) for a, b_ in zip(g0, g1))
        assert not g1[1].requires_grad and not g1[2].requires_grad


def test_never_synchronises():
    r, w, b, y = _inputs(64, 512, 40, 48, torch.float16, True, seed=8)
    for lt in LOSS_TYPES:
        decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=lt)   # first calls: kernel attributes, modules
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for lt in LOSS_TYPES:
            decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=lt)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_target_on_the_cpu_is_rejected():
    r, w, b, y = _inputs(8, 16, 16, 16, torch.float16, True, seed=4)
    with pytest.raises(ValueError, match="must be CUDA tensors on one device"):
        decoded_feature_map_loss_and_grads(r, w, y.cpu(), bias=b)
    with pytest.raises(ValueError, match="must be CUDA tensors on one device"):
        decoded_feature_map_loss_and_grads(r, w, y, bias=b.cpu())


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
def test_k4_view_is_reproducible_and_allocates_only_the_render_gradient_and_workspace(loss_type):
    C, c, H, W = 512, 64, 968, 1296
    g = torch.Generator(device=DEV).manual_seed(9)
    r = torch.randn((c, H, W), generator=g, device=DEV)
    w = torch.randn((C, c), generator=g, device=DEV) / c ** 0.5
    b = 0.1 * torch.randn(C, generator=g, device=DEV)
    y = torch.randn((C, H, W), generator=g, device=DEV, dtype=torch.float16)
    y[:, :40] = 0
    first = decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=loss_type)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    second = decoded_feature_map_loss_and_grads(r, w, y, bias=b, loss_type=loss_type)
    torch.cuda.synchronize()
    ws = _lib.load().sgb_decoded_feature_loss_workspace_bytes(C, c, H * W)
    small = 4 * (w.numel() + b.numel()) + 16               # dL/dW, dL/db and the loss pair
    extra = torch.cuda.max_memory_allocated() - base - 4 * r.numel() - ws
    # the caching allocator hands out a cached large block whole when less than 1 MiB of it would remain
    assert extra <= small + (1 << 20) + (64 << 10), (extra, ws)
    assert float(first[0]) == float(second[0])
    for a, b_ in zip(first[1:], second[1:]):
        assert torch.equal(a, b_)


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


class Cam:
    pass


def _scene(c):
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    scene = make_scene(20000, seed=12, channels=c, scale_mean=0.03)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=DEV)
    pc.active_sh_degree = 0
    cam = orbit_cameras(3, 320, 240)[1]
    v = Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = cam.image_width, cam.image_height, cam.FoVx, cam.FoVy
    v.world_view_transform = torch.as_tensor(cam.world_view_transform, device=DEV)
    v.full_proj_transform = torch.as_tensor(cam.full_proj_transform, device=DEV)
    v.camera_center = torch.as_tensor(cam.camera_center, device=DEV)
    return pc, torch.as_tensor(scene.features, device=DEV), v


def test_compact_field_fit_through_render_chn():
    """Fit a 64-channel field and an nn.Linear(64, 512) decoder with Adam to a 512-channel fp16 feature map rendered
    from a random ground-truth field of the same scene (random 64-channel features through a random 64 -> 512 map, so
    that the compact model can represent it), at the map's size: the cosine loss falls by a clear margin."""
    from semantic_gaussians_b200.renderer import render_chn
    c, C = 64, 512
    pc, feats0, v = _scene(c)
    img_dim = [256, 192]
    g = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
        truth = torch.randn((feats0.shape[0], c), generator=g, device=DEV) @ torch.randn((c, C), generator=g, device=DEV)
        fmap = render_chn(v, pc, Pipe, torch.zeros(C, device=DEV), num_channels=C, override_color=truth,
                          override_shape=img_dim)["render"].half()
    feats = feats0.clone().requires_grad_(True)
    decoder = torch.nn.Linear(c, C, device=DEV)
    opt = torch.optim.Adam([{"params": [feats], "lr": 0.05}, {"params": decoder.parameters(), "lr": 0.01}])
    bg = torch.zeros(c, device=DEV)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        out = render_chn(v, pc, Pipe, bg, num_channels=c, override_color=feats, override_shape=img_dim)
        loss, g_render, g_weight, g_bias = decoded_feature_map_loss_and_grads(out["render"], decoder.weight, fmap,
                                                                              bias=decoder.bias)
        out["render"].backward(g_render)
        decoder.weight.grad, decoder.bias.grad = g_weight, g_bias
        opt.step()
        losses.append(float(loss))
    print(f"compact field fit: cosine loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert losses[-1] < 0.5 * losses[0], losses
