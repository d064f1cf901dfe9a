"""CPU: the timing tools under tools/ and the harness they share (tools/timing.py).  Every tool with an argument parser
starts (`--help` exits 0, so its imports resolve), refuses to run without a CUDA device with its own message, and
card() falls back to a fixed string when nvidia-smi fails."""
import ast
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")

NO_GPU_MESSAGE = {
    "time_adam.py": "time_adam.py needs a GPU",
    "time_decoder_loss.py": "time_decoder_loss.py needs a GPU",
    "time_depth.py": "time_depth.py needs a GPU",
    "time_distill.py": "time_distill.py measures the GPU path and needs a GPU",
    "time_distill_half.py": "time_distill_half.py measures the GPU path and needs a GPU",
    "time_eval.py": "time_eval.py needs a GPU",
    "time_feature_loss.py": "time_feature_loss.py needs a GPU",
    "time_lift.py": "time_lift.py needs a GPU",
    "time_loss.py": "time_loss.py needs a GPU",
    "time_mink_unet.py": "time_mink_unet.py needs a CUDA device",
    "time_voxelize.py": "time_voxelize.py needs a GPU",
}


def _run(script, *args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")      # no device, on any machine
    return subprocess.run([sys.executable, os.path.join(TOOLS, script), *args], capture_output=True, text=True,
                          timeout=300, env=env, cwd=ROOT)


def _timing():
    spec = importlib.util.spec_from_file_location("tools_timing", os.path.join(TOOLS, "timing.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("script", sorted(NO_GPU_MESSAGE))
def test_help_exits_zero(script):
    p = _run(script, "--help")
    assert p.returncode == 0, p.stderr[-2000:]
    assert "usage:" in p.stdout


@pytest.mark.parametrize("script", sorted(NO_GPU_MESSAGE))
def test_refuses_to_run_without_a_gpu(script):
    p = _run(script)
    assert p.returncode != 0
    assert p.stderr.strip().splitlines()[-1] == NO_GPU_MESSAGE[script], p.stderr[-2000:]


def test_time_semantic_compiles_and_its_timing_imports_exist():
    path = os.path.join(TOOLS, "time_semantic.py")
    with open(path) as f:
        source = f.read()
    compile(source, path, "exec")
    timing = _timing()
    names = [a.name for node in ast.walk(ast.parse(source))
             if isinstance(node, ast.ImportFrom) and node.module == "timing" for a in node.names]
    assert names
    for name in names:
        assert hasattr(timing, name), name


@pytest.mark.parametrize("returncode,stdout,want", [
    (0, "NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n", "NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz"),
    (9, "", "unknown (nvidia-smi failed)"),
    (0, "\n", "unknown (nvidia-smi failed)"),
])
def test_card_reads_nvidia_smi_or_falls_back(monkeypatch, returncode, stdout, want):
    timing = _timing()
    seen = []

    def fake_run(cmd, **kw):
        seen.append(cmd)
        return subprocess.CompletedProcess(cmd, returncode, stdout=stdout, stderr="")

    monkeypatch.setattr(timing.subprocess, "run", fake_run)
    assert timing.card() == want
    assert seen == [["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]]
