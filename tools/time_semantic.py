"""Semantic head timings at K3 sizes (256-ch 1080p feature image, K = 21 classes) on one GPU:
  (a) the reference's torch expressions on the rendered image (eval_segmentation.py:155-157),
  (b) sgb_semantic_head on the same image (one pass),
  (c) full pipeline per view: render_chn(256 ch) + head   vs   render_semantic_labels (logit-space render)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from timing import Pipe, device_views, time_ms
from semantic_gaussians_b200.gaussian_model import GaussianModel
from semantic_gaussians_b200.renderer import render_chn
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
from semantic_gaussians_b200.semantic import feature_logits, render_semantic_labels, semantic_head

dev = torch.device("cuda:0")
P, C, K, W, H = 1000000, 256, 21, 1920, 1080
scene = make_scene(P, seed=0, channels=C)
pc = GaussianModel.from_activated(scene.xyz, scene.scales, scene.rotations, scene.opacity, device=dev)
pc.active_sh_degree = 0
feats = torch.as_tensor(scene.features, device=dev).contiguous()
text = torch.nn.functional.normalize(torch.randn(K, C, device=dev), dim=1)
bg = torch.zeros(C, device=dev)
cams = device_views(orbit_cameras(8, W, H), dev)


def rep_ms(fn, reps=10, warm=3):
    """time_ms of fn(i): i = 0..warm-1 in the warm-up, then 0..reps-1 in the timed window."""
    i = iter([*range(warm), *range(reps)])
    return time_ms(lambda: fn(next(i)), reps, warm)


with torch.no_grad():
    imgs = [render_chn(cams[i], pc, Pipe, bg, num_channels=C, override_color=feats)["render"] for i in range(2)]

    def ref_head(i):
        rendering = imgs[i % 2]
        rendering = rendering / (rendering.norm(dim=0, keepdim=True) + 1e-8)
        sim = torch.einsum("cq,qhw->chw", text, rendering)
        return sim[1:].argmax(dim=0)

    t_ref = rep_ms(ref_head)
    t_ours = rep_ms(lambda i: semantic_head(imgs[i % 2], text))
    t_label = rep_ms(lambda i: semantic_head(imgs[i % 2], text, return_sim=False))
    gb = C * W * H * 4 / 1e9
    print(f"head on (256,1080,1920): torch expressions {t_ref:.3f} ms | sgb_semantic_head sim+label {t_ours:.3f} ms "
          f"({gb / t_ours * 1e3:.0f} GB/s of image read) | label only {t_label:.3f} ms ({gb / t_label * 1e3:.0f} GB/s)", flush=True)
    a = ref_head(0); s, l = semantic_head(imgs[0], text)
    print("label agreement with torch:", float((a == l).float().mean()), flush=True)
    del imgs
    t_logits = rep_ms(lambda i: feature_logits(feats, text, pad_to=4))
    print(f"feature_logits (1M x 256 -> 24): {t_logits:.3f} ms ({P * C * 4 / 1e9 / t_logits * 1e3:.0f} GB/s)", flush=True)

    def full(i):
        r = render_chn(cams[i % 8], pc, Pipe, bg, num_channels=C, override_color=feats)["render"]
        return semantic_head(r, text, return_sim=False)[1]

    def full_torch(i):
        rendering = render_chn(cams[i % 8], pc, Pipe, bg, num_channels=C, override_color=feats)["render"]
        rendering = rendering / (rendering.norm(dim=0, keepdim=True) + 1e-8)
        sim = torch.einsum("cq,qhw->chw", text, rendering)
        return sim[1:].argmax(dim=0)

    def fused(i):
        return render_semantic_labels(cams[i % 8], pc, Pipe, bg, text, features=feats)["label"]

    g = feature_logits(feats, text, pad_to=4)

    def fused_pre(i):
        return render_semantic_labels(cams[i % 8], pc, Pipe, bg, text, logits=g)["label"]

    t_ft, t_full, t_fused, t_pre = rep_ms(full_torch), rep_ms(full), rep_ms(fused), rep_ms(fused_pre)
    print(f"label map per view: render_chn + torch head {t_ft:.3f} ms | render_chn + sgb head {t_full:.3f} ms | "
          f"logit-space render {t_fused:.3f} ms | with per-scene logits {t_pre:.3f} ms", flush=True)
    la, lb = full(0), fused(0)
    print("label agreement fused vs full:", float((la == lb).float().mean()), flush=True)
