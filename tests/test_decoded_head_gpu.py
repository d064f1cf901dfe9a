"""Semantic head of a compact field through its linear decoder (semantic.decoded_semantic_head,
semantic.decoded_feature_logits; csrc/decoded_head.cu) on the GPU: similarities and labels against a float64
restatement (decode, normalise, dot with the text, arg-max) with a tolerance scaled by each pixel's condition number,
at every compact width, decoded width and class count the kernels branch on; cross-checks against semantic_head on
the decoded image; per-Gaussian logits; the decoded label render through render_semantic_labels; synchronisation,
reproducibility and memory at a 968 x 1296 view; edge cases."""
import pytest
import torch

from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200.semantic import (decoded_feature_logits, decoded_semantic_head, render_semantic_labels,
                                              semantic_head)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _inputs(c, C, K, H, W, bias, seed, rel=1e-3):
    """render (c,H,W) with some all-zero pixels, weight (C,c), unit text rows (K,C), bias (C) or None.  With a bias,
    b = -W r0 + delta for a random r0 and a delta of ``rel`` times W r0, and a tenth of the pixels are r0 (plus
    zero-pixels): there the decoded pixel is ~rel of its terms (condition number ~1 / rel), where a norm taken as an fp32
    quadratic form loses about 2 log10(1 / rel) of fp32's digits."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = torch.randn((c, H, W), generator=g, device=DEV) * torch.rand((1, H, W), generator=g, device=DEV).add_(0.1)
    w = torch.randn((C, c), generator=g, device=DEV) / c ** 0.5
    t = torch.nn.functional.normalize(torch.randn((K, C), generator=g, device=DEV), dim=1)
    u = torch.rand((H, W), generator=g, device=DEV)
    b = None
    if bias:
        r0 = torch.randn(c, generator=g, device=DEV)
        x0 = w.double() @ r0.double()
        delta = torch.randn(C, generator=g, device=DEV).double() * (rel * x0.norm() / max(C, 1) ** 0.5)
        b = (-x0 + delta).float()
        r[:, u > 0.9] = r0[:, None]
    r[:, u < 0.05] = 0
    if H * W:
        r[:, 0, 0] = 0
    return r.contiguous(), w, t, b


def _reference(r, w, t, b):
    """float64 from the fp32 inputs: (sim64 (K,N), numerators (K,N), kappa (N))."""
    c, H, W = r.shape
    r64 = r.double().reshape(c, -1)
    x = w.double() @ r64
    a = w.double().abs() @ r64.abs()
    if b is not None:
        x += b.double()[:, None]
        a += b.double().abs()[:, None]
    n = x.norm(dim=0)
    num = t.double() @ x
    sim = num / (n + 1e-8)
    an = a.norm(dim=0)
    kappa = torch.where(an > 0, an / n, torch.ones_like(an))      # x = 0 only where every term is 0 -> kappa 1
    return sim, num, kappa


def _check_labels(label, sim64, kappa, first_class):
    s = sim64[first_class:]
    K = s.shape[0]
    want = s.argmax(dim=0)
    if K > 1:
        top2 = s.topk(2, dim=0).values
        clear = (top2[0] - top2[1]) > 1e-4 * kappa.clamp(min=1)
    else:
        clear = torch.ones_like(want, dtype=torch.bool)
    got = label.reshape(-1)
    assert torch.equal(got[clear], want[clear]), f"{int((got[clear] != want[clear]).sum())} clear labels differ"
    assert bool(((got >= 0) & (got < K)).all())
    return clear


CASES = [  # c, C, K, first_class, bias, H, W
    (1, 1, 2, 0, False, 17, 13),
    (1, 5, 21, 1, True, 31, 33),
    (3, 5, 2, 1, True, 40, 37),
    (3, 64, 33, 0, False, 333, 211),
    (16, 64, 21, 1, True, 333, 211),
    (16, 1024, 201, 0, True, 64, 96),
    (64, 512, 21, 1, True, 333, 211),
    (64, 768, 201, 1, False, 128, 128),
    (100, 512, 33, 0, True, 97, 101),
    (100, 1, 2, 1, True, 45, 23),
    (128, 768, 201, 1, True, 96, 130),
    (128, 1024, 33, 0, False, 61, 67),
    (128, 5, 21, 0, True, 333, 211),
    (64, 64, 2, 0, False, 1, 1),
]


@pytest.mark.parametrize("c,C,K,first_class,bias,H,W", CASES)
def test_accuracy_against_float64(c, C, K, first_class, bias, H, W):
    r, w, t, b = _inputs(c, C, K, H, W, bias, seed=c * 1000 + C + K)
    sim, label = decoded_semantic_head(r, w, t, bias=b, first_class=first_class)
    assert sim.shape == (K, H, W) and sim.dtype == torch.float32 and label.shape == (H, W) and label.dtype == torch.int64
    sim64, _, kappa = _reference(r, w, t, b)
    err = (sim.double().reshape(K, -1) - sim64).abs()
    tol = 1e-5 * kappa.clamp(min=1)
    assert bool((err <= tol).all()), f"max err / tol {float((err / tol).max()):.3g}"
    if bias:
        assert float(kappa.max()) > 300          # the ill-conditioned pixels are there
    clear = _check_labels(label, sim64, kappa, first_class)
    if K - first_class > 1 and C > 1 and H * W > 1:               # C = 1: every class is +-1 times x, ties
        assert float(clear.float().mean()) > 0.5
    _, label_only = decoded_semantic_head(r, w, t, bias=b, first_class=first_class, return_sim=False)
    assert torch.equal(label_only, label)


def test_fp32_gram_norm_fails_on_ill_conditioned_pixels():
    """The accuracy test bites: with ||x||^2 as an fp32 quadratic form the similarities of pixels with a condition
    number ~1e5 miss the tolerance; the float64 form meets it there."""
    r, w, t, b = _inputs(64, 512, 21, 64, 64, True, seed=5, rel=1e-5)
    sim64, num64, kappa = _reference(r, w, t, b)
    r2 = r.reshape(64, -1)
    G, u, bb = w.T @ w, w.T @ b, b @ b
    q = (r2 * (G @ r2)).sum(0) + 2 * (u @ r2) + bb
    sim32 = num64.float() / (q.clamp(min=0).sqrt() + 1e-8)
    assert bool(((sim32.double() - sim64).abs() > 1e-5 * kappa.clamp(min=1)).any())
    sim, _ = decoded_semantic_head(r, w, t, bias=b)
    assert bool(((sim.double().reshape(21, -1) - sim64).abs() <= 1e-5 * kappa.clamp(min=1)).all())


def test_identity_decoder_matches_semantic_head():
    g = torch.Generator(device=DEV).manual_seed(3)
    c, K, H, W = 64, 21, 97, 130
    r = torch.randn((c, H, W), generator=g, device=DEV)
    t = torch.nn.functional.normalize(torch.randn((K, c), generator=g, device=DEV), dim=1)
    sim, label = decoded_semantic_head(r, torch.eye(c, device=DEV), t)
    sim_ref, label_ref = semantic_head(r, t)
    assert float((sim - sim_ref).abs().max()) <= 1e-6
    top2 = sim_ref[1:].topk(2, dim=0).values
    clear = (top2[0] - top2[1]) > 1e-4
    assert torch.equal(label[clear], label_ref[clear]) and float(clear.float().mean()) > 0.9


@pytest.mark.parametrize("c,C,K,first_class", [(64, 512, 21, 1), (128, 768, 201, 0), (3, 33, 33, 1)])
def test_matches_semantic_head_on_the_decoded_image(c, C, K, first_class):
    r, w, t, b = _inputs(c, C, K, 120, 97, True, seed=7)
    x = torch.einsum("kc,chw->khw", w, r) + b[:, None, None]
    sim_ref, label_ref = semantic_head(x, t, first_class=first_class)
    sim, label = decoded_semantic_head(r, w, t, bias=b, first_class=first_class)
    sim64, _, kappa = _reference(r, w, t, b)
    tol = 1e-5 * kappa.clamp(min=1).reshape(120, 97)
    assert bool(((sim - sim_ref).abs() <= 2 * tol).all())
    top2 = sim64[first_class:].topk(2, dim=0).values
    clear = ((top2[0] - top2[1]) > 1e-4 * kappa.clamp(min=1)).reshape(120, 97)
    assert torch.equal(label[clear], label_ref[clear])


def test_label_only_call_is_bitwise_the_labels_and_writes_no_planes():
    r, w, t, b = _inputs(64, 512, 201, 133, 171, True, seed=9)
    sim, label = decoded_semantic_head(r, w, t, bias=b)
    none, label_only = decoded_semantic_head(r, w, t, bias=b, return_sim=False)
    assert none is None and torch.equal(label_only, label)
    sim_only, no_label = decoded_semantic_head(r, w, t, bias=b, return_label=False)
    assert no_label is None and torch.equal(sim_only, sim)
    # through the C entry point: a NaN-filled sim buffer next to a label-only call stays untouched
    lib = _lib.load()
    C_, c = w.shape
    K = t.shape[0]
    N = r.shape[1] * r.shape[2]
    ws = torch.empty(lib.sgb_decoded_semantic_head_workspace_bytes(C_, c, K), dtype=torch.uint8, device=DEV)
    guard = torch.full((K, N), float("nan"), device=DEV)
    lab = torch.full((N,), -7, dtype=torch.int64, device=DEV)
    _lib.check(lib.sgb_decoded_semantic_head(C_, c, K, N, r.data_ptr(), w.data_ptr(), b.data_ptr(), t.data_ptr(), 1,
                                             None, lab.data_ptr(), ws.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
    assert torch.equal(lab, label.reshape(-1)) and bool(guard.isnan().all())


@pytest.mark.parametrize("P,c,C,K,pad,bias", [(1, 1, 1, 2, 1, False), (1000, 16, 64, 21, 4, True),
                                              (4097, 64, 512, 201, 4, True), (333, 100, 768, 33, 8, False),
                                              (2048, 128, 1024, 21, 1, True)])
def test_decoded_feature_logits_match_float64(P, c, C, K, pad, bias):
    g = torch.Generator(device=DEV).manual_seed(P + c)
    f = torch.randn((P, c), generator=g, device=DEV)
    w = torch.randn((C, c), generator=g, device=DEV) / c ** 0.5
    t = torch.nn.functional.normalize(torch.randn((K, C), generator=g, device=DEV), dim=1)
    b = 0.3 * torch.randn(C, generator=g, device=DEV) if bias else None
    out = decoded_feature_logits(f, w, t, bias=b, pad_to=pad)
    Kpad = (K + pad - 1) // pad * pad
    assert out.shape == (P, Kpad) and out.dtype == torch.float32
    x = f.double() @ w.double().T + (b.double() if bias else 0)
    want = torch.einsum("cq,dq->dc", t.double(), x)
    scale = (f.double().abs() @ w.double().abs().T + (b.double().abs() if bias else 0)) @ t.double().abs().T
    assert bool(((out[:, :K].double() - want).abs() <= 1e-5 * scale).all())
    assert bool((out[:, K:] == 0).all())


def test_decoded_label_render_matches_render_then_decode():
    """render_semantic_labels on decoded per-Gaussian logits with the background decoded the same way equals
    render_chn(c) -> decode -> semantic_head: the weights and the final transmittance sum to one, so text . b blends
    through.  The view has uncovered pixels (T = 1) and saturated pixels (the early stop at T < 1e-4)."""
    from types import SimpleNamespace

    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.renderer import render_chn
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras

    c, C, K = 16, 512, 21
    scene = make_scene(1_000_000, seed=11, channels=c, scale_mean=0.04)
    keep = (scene.xyz ** 2).sum(1) < 0.7 ** 2              # a dense ball that leaves the view's corners uncovered
    pc = GaussianModel.from_activated(scene.xyz[keep], scene.scales[keep], scene.rotations[keep], scene.opacity[keep],
                                      device=DEV)
    pc.active_sh_degree = 0
    g = torch.Generator(device=DEV).manual_seed(4)
    f = torch.as_tensor(scene.features[keep], device=DEV).contiguous()
    w = torch.randn((C, c), generator=g, device=DEV) / c ** 0.5
    b = 0.5 * torch.randn(C, generator=g, device=DEV)
    t = torch.nn.functional.normalize(torch.randn((K, C), generator=g, device=DEV), dim=1)
    bg_c = torch.full((c,), 0.3, device=DEV)
    pipe = SimpleNamespace(convert_shs_python=False, compute_cov3d_python=False, debug=False)
    cam = orbit_cameras(3, 320, 240)[1]
    v = SimpleNamespace(image_width=cam.image_width, image_height=cam.image_height, FoVx=cam.FoVx, FoVy=cam.FoVy,
                        world_view_transform=torch.as_tensor(cam.world_view_transform, device=DEV),
                        full_proj_transform=torch.as_tensor(cam.full_proj_transform, device=DEV),
                        camera_center=torch.as_tensor(cam.camera_center, device=DEV))

    # coverage: an all-ones field renders 1 - T, so uncovered and saturated pixels are both present
    with torch.no_grad():
        cover = render_chn(v, pc, pipe, torch.zeros(1, device=DEV), num_channels=1,
                           override_color=torch.ones((f.shape[0], 1), device=DEV))["render"][0]
    assert bool((cover == 0).any()), "no uncovered pixel in the view"
    assert bool((cover > 1 - 1e-4).any()), "no saturated pixel in the view"

    with torch.no_grad():
        r = render_chn(v, pc, pipe, bg_c, num_channels=c, override_color=f)["render"]
    x = torch.einsum("kc,chw->khw", w.double(), r.double()) + b.double()[:, None, None]
    raw = torch.einsum("kc,chw->khw", t.double(), x)
    sim_ref, label_ref = semantic_head(x.float(), t)
    out = render_semantic_labels(v, pc, pipe, w @ bg_c + b, t, logits=decoded_feature_logits(f, w, t, b, pad_to=4))
    assert out["logits"].shape == raw.shape
    assert float((out["logits"].double() - raw).abs().max()) <= 1e-4 * float(raw.abs().max())
    top2 = raw[1:].topk(2, dim=0).values
    clear = (top2[0] - top2[1]) > 1e-4 * float(raw.abs().max())
    assert float(clear.float().mean()) > 0.9
    assert torch.equal(out["label"][clear], label_ref[clear])
    # the decoded head on the c-channel render gives the same labels
    _, label_c = decoded_semantic_head(r, w, t, bias=b, return_sim=False)
    assert torch.equal(label_c[clear], label_ref[clear])


def test_no_sync_reproducible_and_memory_bounded_at_view_size():
    c, C, K, H, W = 64, 512, 21, 968, 1296
    r, w, t, b = _inputs(c, C, K, H, W, True, seed=1)
    decoded_semantic_head(r, w, t, bias=b)                        # load the library, set kernel attributes
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        s1, l1 = decoded_semantic_head(r, w, t, bias=b)
        s2, l2 = decoded_semantic_head(r, w, t, bias=b)
        _, l3 = decoded_semantic_head(r, w, t, bias=b, return_sim=False)
        f = torch.randn((100_000, c), device=DEV)
        o1 = decoded_feature_logits(f, w, t, b, pad_to=4)
        o2 = decoded_feature_logits(f, w, t, b, pad_to=4)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(s1, s2) and torch.equal(l1, l2) and torch.equal(l1, l3) and torch.equal(o1, o2)
    del s1, s2, l1, l2, l3
    ws = _lib.load().sgb_decoded_semantic_head_workspace_bytes(C, c, K)
    for return_sim in (True, False):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = decoded_semantic_head(r, w, t, bias=b, return_sim=return_sim)
        torch.cuda.synchronize()
        outputs = (K * H * W * 4 if return_sim else 0) + H * W * 8
        peak = torch.cuda.max_memory_allocated() - base
        assert peak <= outputs + ws + 4096, (peak, outputs, ws)
        assert peak < outputs + C * H * W * 4 // 8
        del out


def test_empty_image_and_empty_table():
    r, w, t, b = _inputs(16, 64, 21, 0, 5, True, seed=2)
    sim, label = decoded_semantic_head(r, w, t, bias=b)
    assert sim.shape == (21, 0, 5) and label.shape == (0, 5)
    out = decoded_feature_logits(torch.empty((0, 16), device=DEV), w, t, b, pad_to=4)
    assert out.shape == (0, 24)


def test_non_contiguous_inputs():
    r, w, t, b = _inputs(32, 96, 33, 50, 60, True, seed=6)
    want_sim, want_label = decoded_semantic_head(r, w, t, bias=b)
    rn = r.permute(0, 2, 1).contiguous().permute(0, 2, 1)        # (c,H,W) view with transposed strides
    wn = w.T.contiguous().T
    tn = torch.cat([t, t], dim=1)[:, ::2]
    tn.copy_(t)
    bn = torch.stack([b, b], dim=1)[:, 0]
    assert not (rn.is_contiguous() or wn.is_contiguous() or tn.is_contiguous() or bn.is_contiguous())
    sim, label = decoded_semantic_head(rn, wn, tn, bias=bn)
    assert torch.equal(sim, want_sim) and torch.equal(label, want_label)
    f = torch.randn((300, 64), device=DEV)[:, ::2]
    assert torch.equal(decoded_feature_logits(f, wn, tn, bn, pad_to=4),
                       decoded_feature_logits(f.contiguous(), w, t, b, pad_to=4))


def test_cpu_tensor_is_rejected():
    r, w, t, b = _inputs(8, 16, 5, 10, 10, True, seed=8)
    with pytest.raises(ValueError, match="CUDA tensors on one device"):
        decoded_semantic_head(r.cpu(), w, t, bias=b)
    with pytest.raises(ValueError, match="CUDA tensors on one device"):
        decoded_semantic_head(r, w, t, bias=b.cpu())
    with pytest.raises(ValueError, match="CUDA tensors on one device"):
        decoded_feature_logits(torch.randn((4, 8)), w, t, b)
