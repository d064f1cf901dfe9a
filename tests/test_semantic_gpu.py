"""GPU parity of the semantic head against the numpy oracle and against the reference's
torch expressions, plus the logit-space label renderer against render_chn + head."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pytestmark = pytest.mark.gpu


def _case(C, K, H, W, seed):
    rng = np.random.default_rng(seed)
    r = rng.standard_normal((C, H, W)).astype(np.float32) * rng.uniform(0.1, 3.0, (1, H, W)).astype(np.float32)
    t = rng.standard_normal((K, C)).astype(np.float32)
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    return r, t


@pytest.mark.parametrize("C,K,H,W,first", [
    (16, 5, 7, 9, 1),        # ragged: H*W % 4 != 0 -> scalar pixel path
    (64, 21, 32, 48, 1),     # ScanNet-20 + "other"
    (256, 21, 60, 80, 1),
    (256, 21, 50, 82, 1),    # last 1024-pixel block partial (4100 px)
    (768, 21, 16, 64, 1),    # OpenSeg width
    (768, 29, 16, 64, 1),    # ring + 32-class embedding table at the shared-memory limit
    (130, 8, 16, 20, 0),     # C not a multiple of the 128-channel slab, first_class 0
    (40, 3, 8, 8, 2),        # single candidate class
    (48, 41, 16, 16, 1),     # K > 32: two class passes
    (48, 70, 12, 12, 35),    # K > 32 and first_class inside the second pass
])
def test_head_matches_oracle(C, K, H, W, first):
    from oracle import semantic_oracle as so
    from semantic_gaussians_b200.semantic import semantic_head
    r, t = _case(C, K, H, W, C * 1000 + K)
    r[:, 0, 0] = 0.0                                      # an empty pixel: sim 0 everywhere, label 0
    dev = torch.device("cuda:0")
    sim, label = semantic_head(torch.from_numpy(r).to(dev), torch.from_numpy(t).to(dev), first_class=first)
    osim, olabel = so.semantic_head(r, t, first)
    sim, label = sim.cpu().numpy(), label.cpu().numpy()
    assert label.dtype == np.int64 and sim.shape == osim.shape
    assert np.abs(sim - osim).max() <= 1e-4 * np.abs(osim).max() + 1e-6       # 1e-4 rel fp32
    assert np.all(sim[:, 0, 0] == 0.0) and label[0, 0] == 0
    clear = so.label_margin(osim, first) > 1e-5
    assert np.array_equal(label[clear], olabel[clear])
    # label-only and sim-only calls give the same answers
    _, l2 = semantic_head(torch.from_numpy(r).to(dev), torch.from_numpy(t).to(dev), first_class=first, return_sim=False)
    s2, n2 = semantic_head(torch.from_numpy(r).to(dev), torch.from_numpy(t).to(dev), first_class=first, return_label=False)
    assert n2 is None and np.array_equal(l2.cpu().numpy(), label) and np.array_equal(s2.cpu().numpy(), sim)


def test_head_matches_reference_torch_expressions():
    from semantic_gaussians_b200.semantic import semantic_head
    r, t = _case(192, 21, 96, 128, 7)
    dev = torch.device("cuda:0")
    rendering, text_features = torch.from_numpy(r).to(dev), torch.from_numpy(t).to(dev)
    sim, label = semantic_head(rendering, text_features)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        rn = rendering / (rendering.norm(dim=0, keepdim=True) + 1e-8)        # eval_segmentation.py:155
        ref = torch.einsum("cq,qhw->chw", text_features, rn)                  # :156
        ref_label = ref[1:].argmax(dim=0)                                     # :157
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    assert float((sim - ref).abs().max()) <= 1e-4 * float(ref.abs().max())
    top2 = ref[1:].topk(2, dim=0).values
    clear = (top2[0] - top2[1]) > 1e-5
    assert bool(clear.float().mean() > 0.95) and torch.equal(label[clear], ref_label[clear])


@pytest.mark.parametrize("P,C,K,pad", [(1000, 24, 7, 1), (5000, 256, 21, 4), (777, 130, 40, 4), (64, 768, 21, 4)])
def test_feature_logits_match_oracle(P, C, K, pad):
    from oracle import semantic_oracle as so
    from semantic_gaussians_b200.semantic import feature_logits
    rng = np.random.default_rng(P + C)
    f = rng.standard_normal((P, C)).astype(np.float32)
    t = rng.standard_normal((K, C)).astype(np.float32)
    dev = torch.device("cuda:0")
    g = feature_logits(torch.from_numpy(f).to(dev), torch.from_numpy(t).to(dev), pad_to=pad).cpu().numpy()
    Kpad = (K + pad - 1) // pad * pad
    o = so.feature_logits(f, t)
    assert g.shape == (P, Kpad) and np.all(g[:, K:] == 0.0)
    assert np.abs(g[:, :K] - o).max() <= 1e-4 * np.abs(o).max()


def test_label_argmax_matches_torch():
    from semantic_gaussians_b200.semantic import label_argmax
    dev = torch.device("cuda:0")
    planes = torch.randn((24, 37, 53), device=dev)
    assert torch.equal(label_argmax(planes, 21, 1), planes[1:21].argmax(dim=0))
    assert torch.equal(label_argmax(planes, None, 0), planes.argmax(dim=0))


def test_logit_space_labels_match_feature_image_head():
    """render_semantic_labels (K-channel logit render) == render_chn(C channels) -> semantic_head, where the
    class margin is above fp32 noise; un-normalised logits agree to 1e-4 rel."""
    from semantic_gaussians_b200.gaussian_model import GaussianModel
    from semantic_gaussians_b200.renderer import render_chn
    from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
    from semantic_gaussians_b200.semantic import render_semantic_labels, semantic_head
    dev = torch.device("cuda:0")
    C, K = 64, 21
    scene = make_scene(20000, seed=11, channels=C)
    pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
    pc.active_sh_degree = 0
    feats = torch.as_tensor(scene.features, device=dev).contiguous()
    text = torch.nn.functional.normalize(torch.randn(K, C, device=dev), dim=1)
    bg = torch.full((C,), 0.05, device=dev)

    class Pipe:
        convert_shs_python = False
        compute_cov3d_python = False
        debug = False

    class Cam:
        pass

    c = orbit_cameras(3, 320, 240)[1]
    v = Cam()
    v.image_width, v.image_height, v.FoVx, v.FoVy = c.image_width, c.image_height, c.FoVx, c.FoVy
    v.world_view_transform = torch.as_tensor(c.world_view_transform, device=dev)
    v.full_proj_transform = torch.as_tensor(c.full_proj_transform, device=dev)
    v.camera_center = torch.as_tensor(c.camera_center, device=dev)

    full = render_chn(v, pc, Pipe, bg, num_channels=C, override_color=feats)["render"]
    sim, label = semantic_head(full, text)
    raw = torch.einsum("kc,chw->khw", text, full)                 # un-normalised similarities of the full render
    out = render_semantic_labels(v, pc, Pipe, bg, text, features=feats)
    assert out["logits"].shape == raw.shape and out["label"].shape == label.shape
    assert float((out["logits"] - raw).abs().max()) <= 1e-4 * float(raw.abs().max())
    top2 = sim[1:].topk(2, dim=0).values
    clear = (top2[0] - top2[1]) > 1e-4
    assert bool(clear.float().mean() > 0.9) and torch.equal(out["label"][clear], label[clear])
    from semantic_gaussians_b200.semantic import feature_logits
    out2 = render_semantic_labels(v, pc, Pipe, bg, text, logits=feature_logits(feats, text, pad_to=4))
    assert torch.equal(out2["label"], out["label"]) and torch.equal(out2["logits"], out["logits"])


@pytest.mark.parametrize("C,K,H,W,dtype", [(16, 5, 7, 9, torch.int64), (256, 21, 64, 96, torch.int32), (130, 33, 20, 16, torch.int64)])
def test_distill_loss_and_grad(C, K, H, W, dtype):
    from oracle import semantic_oracle as so
    from semantic_gaussians_b200.semantic import distill_loss_and_grad
    dev = torch.device("cuda:0")
    r, t = _case(C, K, H, W, 5 * C + K)
    lab = np.random.default_rng(C).integers(0, K, (H, W))
    R = torch.from_numpy(r).to(dev).requires_grad_(True)
    loss, grad = distill_loss_and_grad(R, torch.from_numpy(t).to(dev), torch.from_numpy(lab).to(dev).to(dtype))
    oloss, ograd = so.distill_loss_and_grad(r, t, lab)
    assert loss.dtype == torch.float64 and abs(float(loss) - oloss) <= 1e-5 * abs(oloss) + 1e-9
    assert np.allclose(grad.cpu().numpy(), ograd, rtol=1e-6, atol=0)
    # same thing through torch autograd (what the e2e bench arm used before)
    tl = -(R * torch.from_numpy(t).to(dev)[torch.from_numpy(lab).to(dev)].permute(2, 0, 1)).mean()
    tl.backward()
    assert abs(float(tl) - float(loss)) <= 1e-4 * abs(float(tl)) + 1e-9
    assert torch.allclose(R.grad, grad, rtol=1e-5, atol=1e-12)
