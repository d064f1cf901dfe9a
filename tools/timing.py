"""The measuring harness the time_*.py tools share: the card a number was taken on, one CUDA-event timer, one
torch.profiler pass, and the renderer's view objects built from scene_synth cameras.

Every timed window is bracketed by device synchronises, so it measures finished work rather than the enqueue, and the
profiler runs in a pass of its own, apart from the timed windows, because tracing slows the host."""
import subprocess
from types import SimpleNamespace

import torch


class Pipe:
    """The pipeline flags render / render_chn read: native SH colour and covariance, no debug checks."""
    convert_shs_python = False
    compute_cov3d_python = False
    debug = False


def card() -> str:
    """Name, power limit and max SM clock of the first GPU, as nvidia-smi reports them."""
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def gpu(tool: str):
    """(cuda:0, card()) after printing the card line; exits with "<tool> needs a GPU" where there is none."""
    if not torch.cuda.is_available():
        raise SystemExit(f"{tool} needs a GPU")
    dev = torch.device("cuda:0")
    name = card()
    print(f"card (name, power limit, max SM clock): {name}", flush=True)
    return dev, name


def time_ms(fn, reps: int = 1, warmup: int = 0) -> float:
    """Mean ms per call of fn() over `reps` calls between two CUDA events, after `warmup` untimed calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, n: int = 1, names=None, warmup: int = 0) -> dict:
    """Device ms per call of the CUDA kernels of `n` calls of fn() under torch.profiler, after `warmup` unprofiled
    calls.  With `names`, {name: ms} summed over the kernels whose name contains it (names no kernel matches are left
    out); without, {kernel name cut to 90 characters: ms}, longest first."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name != "CUDA" or not e.count:
            continue
        ms = e.device_time_total / 1e3 / n
        if names is None:
            out[e.key[:90]] = ms
            continue
        for name in names:
            if name in e.key:
                out[name] = out.get(name, 0.0) + ms
    return out if names is not None else dict(sorted(out.items(), key=lambda kv: -kv[1]))


def device_views(cams, device):
    """The view objects render / render_chn take, one per scene_synth SynthCamera, with its matrices on `device`."""
    return [SimpleNamespace(image_width=c.image_width, image_height=c.image_height, FoVx=c.FoVx, FoVy=c.FoVy,
                            world_view_transform=torch.as_tensor(c.world_view_transform, device=device),
                            full_proj_transform=torch.as_tensor(c.full_proj_transform, device=device),
                            camera_center=torch.as_tensor(c.camera_center, device=device)) for c in cams]
