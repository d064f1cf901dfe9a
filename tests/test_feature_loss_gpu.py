"""Feature-map distillation loss (semantic.feature_map_loss_and_grad, sgb_feature_map_loss) on the GPU: loss, pixel
count and gradient against float64 torch autograd of the reference's expressions (distill.py:111-124) at every
channel count, target dtype and image shape its kernels branch on; reproducibility and memory at K3 size; and a
short feature fit through render_chn."""
import pytest
import torch
from feature_loss_ref import feature_loss

from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200.semantic import feature_map_loss_and_grad

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LOSS_TYPES = ("cosine", "l1", "l2")


def _inputs(C, H, W, dtype, seed):
    """render / target with: target pixels that are all zero, target pixels with a single non-zero (last) channel,
    render pixels with |x| < 1e-8 (one of them exactly zero), and render values equal to the target (|x - y| = 0)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = torch.randn((C, H, W), generator=g, device=DEV) * torch.rand((1, H, W), generator=g, device=DEV).add_(0.1)
    y = (0.6 * r + torch.randn((C, H, W), generator=g, device=DEV)).to(dtype)
    u = torch.rand((H, W), generator=g, device=DEV)
    y[:, u < 0.1] = 0
    if C > 1:
        y[:-1, (u >= 0.1) & (u < 0.15)] = 0
    r[:, (u >= 0.15) & (u < 0.2)] *= 1e-10
    r[:, 0, 0] = 0
    tie = torch.rand((C, H, W), generator=g, device=DEV) < 0.05
    r[tie] = y.float()[tie]
    return r.contiguous(), y.contiguous()


def _reference(r, y, loss_type):
    """feature_loss_ref.feature_loss with one row per pixel: (loss, d loss / d r (C,H,W), pixels averaged over)."""
    C, H, W = r.shape
    loss, n, g = feature_loss(r.permute(1, 2, 0).reshape(-1, C), y.permute(1, 2, 0).reshape(-1, C), loss_type)
    return loss, g.reshape(H, W, C).permute(2, 0, 1), n


def _abi_count(r, y, loss_type):
    """loss[1] of the C entry point: the pixels the mean runs over."""
    out = torch.empty(2, dtype=torch.float64, device=DEV)
    grad = torch.empty_like(r)
    dtype = _lib.FEAT_F16 if y.dtype == torch.float16 else _lib.FEAT_F32
    lt = {"cosine": _lib.FEATLOSS_COSINE, "l1": _lib.FEATLOSS_L1, "l2": _lib.FEATLOSS_L2}[loss_type]
    _lib.check(_lib.load().sgb_feature_map_loss(r.shape[0], r.shape[1] * r.shape[2], r.data_ptr(), y.data_ptr(), dtype,
                                               lt, grad.data_ptr(), out.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
    return out.cpu()


def _check(r, y, loss_type):
    loss, grad = feature_map_loss_and_grad(r, y, loss_type)
    want_loss, want_grad, want_n = _reference(r, y, loss_type)
    assert loss.dtype == torch.float64 and loss.ndim == 0 and loss.is_cuda
    assert grad.dtype == torch.float32 and grad.shape == r.shape
    assert abs(float(loss) - want_loss) <= 1e-5 * abs(want_loss) + 1e-7, (float(loss), want_loss)
    err = (grad.double() - want_grad).abs()
    scale = float(want_grad.abs().max())
    assert float(err.max()) <= 1e-5 * scale, (float(err.max()), scale)
    # the pixels with a clamped render norm have a 1e8-times larger gradient: the rest must match on their own scale,
    # which for cosine is that of the two terms y / (a b) and cos x / (a |x|), each at most 1 / (Nv |x|) (they cancel
    # where x is parallel to y, e.g. everywhere at C = 1)
    xn = r.double().norm(dim=0)
    normal = xn >= 1e-8
    scale_n = float(want_grad[:, normal].abs().max())
    if loss_type == "cosine" and want_n:
        valid = normal & (y.double().norm(dim=0) > 0)
        scale_n = max(scale_n, float((1.0 / (want_n * xn[valid])).max()))
    assert float(err[:, normal].max()) <= 1e-5 * scale_n, (float(err[:, normal].max()), scale_n)
    if loss_type == "l1":  # sign(0) = 0 at the tied values
        assert torch.equal(grad[r == y.float()], torch.zeros_like(grad[r == y.float()]))
    assert _abi_count(r, y, loss_type)[1].item() == want_n


# (C, H, W): planes of N % 8 == 0 pixels take the TMA staging of the cosine kernel, the others plain loads;
# C > 256 needs several TMA boxes (300: two boxes of 160 rows, 20 of them past C); ragged N leaves a partial block.
SHAPES = [
    (1, 37, 250), (1, 64, 64), (3, 64, 64), (5, 333, 211), (5, 40, 48),
    (64, 37, 250), (64, 64, 96), (256, 333, 211), (256, 48, 64), (300, 24, 40),
    (768, 37, 25), (768, 32, 64), (1024, 19, 21), (1024, 16, 40),
]


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("C,H,W", SHAPES)
def test_matches_float64_torch(C, H, W, dtype, loss_type):
    r, y = _inputs(C, H, W, dtype, seed=C * 7 + H)
    _check(r, y, loss_type)


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
def test_matches_float64_torch_at_1080p(dtype, loss_type):
    r, y = _inputs(256, 1080, 1920, dtype, seed=3)
    _check(r, y, loss_type)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("C,H,W", [(64, 37, 250), (256, 48, 64)])
def test_all_zero_target_gives_zero_loss_count_and_gradient(C, H, W, dtype):
    r, _ = _inputs(C, H, W, dtype, seed=1)
    y = torch.zeros((C, H, W), dtype=dtype, device=DEV)
    loss, grad = feature_map_loss_and_grad(r, y)
    assert float(loss) == 0.0 and not bool(grad.any())
    assert _abi_count(r, y, "cosine").tolist() == [0.0, 0.0]


def test_empty_image_and_non_contiguous_inputs():
    loss, grad = feature_map_loss_and_grad(torch.zeros((8, 0, 5), device=DEV), torch.zeros((8, 0, 5), device=DEV).half())
    assert float(loss) == 0.0 and grad.shape == (8, 0, 5)
    r, y = _inputs(16, 40, 24, torch.float16, seed=2)
    for lt in LOSS_TYPES:
        l0, g0 = feature_map_loss_and_grad(r, y, lt)
        rt, yt = r.transpose(1, 2).contiguous().transpose(1, 2), y.transpose(1, 2).contiguous().transpose(1, 2)
        assert not rt.is_contiguous() and not yt.is_contiguous()
        l1, g1 = feature_map_loss_and_grad(rt, yt, lt)
        assert float(l0) == pytest.approx(float(l1), rel=1e-12) and torch.equal(g0, g1)


def test_never_synchronises():
    r, y = _inputs(64, 40, 48, torch.float16, seed=8)
    for lt in LOSS_TYPES:
        feature_map_loss_and_grad(r, y, lt)            # first calls: kernel attributes and module loading
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for lt in LOSS_TYPES:
            feature_map_loss_and_grad(r, y, lt)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_target_on_the_cpu_is_rejected():
    r, y = _inputs(8, 16, 16, torch.float16, seed=4)
    with pytest.raises(ValueError, match="must be CUDA tensors on one device"):
        feature_map_loss_and_grad(r, y.cpu())


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
def test_k3_size_is_reproducible_and_allocates_only_the_gradient(loss_type):
    r, y = _inputs(256, 1080, 1920, torch.float16, seed=9)
    _, g0 = feature_map_loss_and_grad(r, y, loss_type)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss, g1 = feature_map_loss_and_grad(r, y, loss_type)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - g1.numel() * 4
    assert extra <= 4 << 20, extra
    assert torch.equal(g0, g1)


class Pipe:
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


class Cam:
    pass


def _scene(C):
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    scene = make_scene(20000, seed=12, channels=C, scale_mean=0.03)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=DEV)
    pc.active_sh_degree = 0
    c = orbit_cameras(3, 320, 240)[1]
    v = Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
    v.world_view_transform = torch.as_tensor(c.world_view_transform, device=DEV)
    v.full_proj_transform = torch.as_tensor(c.full_proj_transform, device=DEV)
    v.camera_center = torch.as_tensor(c.camera_center, device=DEV)
    return pc, torch.as_tensor(scene.features, device=DEV), v


@pytest.mark.parametrize("loss_type", LOSS_TYPES)
def test_feature_fit_through_render_chn(loss_type):
    """Fit (P, 64) features to an fp16 feature map rendered from other features of the same scene, at the map's
    size (override_shape): the loss falls by a clear margin within a few dozen Adam steps."""
    from semantic_gaussians_b200.renderer import render_chn
    C = 64
    pc, feats0, v = _scene(C)
    img_dim = [256, 192]                                   # (w, h) of the 2D feature map
    bg = torch.zeros(C, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
        other = torch.randn(feats0.shape, generator=g, device=DEV)
        fmap = render_chn(v, pc, Pipe, bg, num_channels=C, override_color=other, override_shape=img_dim)["render"]
        fmap = fmap.half()
    feats = feats0.clone().requires_grad_(True)
    opt = torch.optim.Adam([feats], lr=0.05)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        out = render_chn(v, pc, Pipe, bg, num_channels=C, override_color=feats, override_shape=img_dim)
        loss, grad = feature_map_loss_and_grad(out["render"], fmap, loss_type)
        out["render"].backward(grad)
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.5 * losses[0], losses


def test_feature_gradient_equals_torch_autograd_of_the_cosine_expression():
    from semantic_gaussians_b200.renderer import render_chn
    C = 64
    pc, feats0, v = _scene(C)
    img_dim = [256, 192]
    bg = torch.zeros(C, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(6)
    with torch.no_grad():
        other = torch.randn(feats0.shape, generator=g, device=DEV)
        fmap = render_chn(v, pc, Pipe, bg, num_channels=C, override_color=other, override_shape=img_dim)["render"].half()
    feats = feats0.clone().requires_grad_(True)
    out = render_chn(v, pc, Pipe, bg, num_channels=C, override_color=feats, override_shape=img_dim)["render"]
    loss, grad = feature_map_loss_and_grad(out, fmap)
    out.backward(grad, retain_graph=True)
    fused = feats.grad.clone()
    feats.grad = None
    t = fmap.float()
    m = t.norm(dim=0) > 0
    tl = (1 - torch.nn.functional.cosine_similarity(out, t, dim=0))[m].mean()
    tl.backward()
    assert abs(float(tl.detach()) - float(loss)) <= 1e-5 * abs(float(tl.detach())) + 1e-7
    scale = float(feats.grad.abs().max())
    assert scale > 0 and float((fused - feats.grad).abs().max()) <= 1e-4 * scale
