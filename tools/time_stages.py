"""Stage timings (library tracing) of one C-channel forward + backward workload.
usage: python tools/time_stages.py [P W H C reps]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from semantic_gaussians_b200 import _lib
from semantic_gaussians_b200.scene_synth import make_scene, orbit_cameras
from util import dev_cam, dev_scene, run_ours

P, W, H, C, reps = (int(x) for x in (sys.argv[1:6] + ["1000000", "1920", "1080", "256", "5"][len(sys.argv) - 1:]))
dev = torch.device("cuda:0")
scene = make_scene(P, 0, channels=C)
cams = orbit_cameras(8, W, H)
sc = dev_scene(scene, dev, requires_grad=True)
bg = torch.zeros(C, device=dev)
dL = torch.randn((C, H, W), device=dev) / (H * W)
ctx = _lib.ctx_for(0, torch.cuda.current_stream(dev).cuda_stream)


def step(i):
    o = run_ours("chn", sc, dev_cam(cams[i % 8], dev), bg, use_features=True)
    o["color"].backward(dL)
    for v in sc.values():
        if v is not None:
            v.grad = None


for i in range(2):
    step(i)
torch.cuda.synchronize()
_lib.profile_enable(ctx, True)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(reps):
    step(i)
e1.record()
torch.cuda.synchronize()
st = _lib.profile_read(ctx)
_lib.profile_enable(ctx, False)
print(f"total {e0.elapsed_time(e1) / reps:.3f} ms/step |",
      " ".join(f"{k}={v[0] / max(v[1], 1):.3f}" for k, v in st.items() if v[1]), flush=True)
