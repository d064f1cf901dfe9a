"""Decoded semantic head without a GPU: the symbols are bound, sgb_decoded_semantic_head and sgb_decoded_feature_logits
reject every bad argument before anything is enqueued, the workspace depends on the widths only, the Python layer
raises ValueError for bad tensors, and tools/time_decoded_semantic.py parses its arguments and refuses to run without
a device."""
import os
import subprocess
import sys

import pytest
import torch

from semantic_gaussians_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _head(lib, C=8, c=4, K=5, N=64, render=1, weight=1, bias=None, text=1, first_class=1, sim=1, label=8, ws=256):
    return lib.sgb_decoded_semantic_head(C, c, K, N, render, weight, bias, text, first_class, sim, label, ws, None)


def _logits(lib, P=10, C=8, c=4, K=5, Kpad=8, features=1, weight=1, bias=None, text=1, out=1, ws=256):
    return lib.sgb_decoded_feature_logits(P, C, c, K, Kpad, features, weight, bias, text, out, ws, None)


def test_symbols_are_bound():
    lib = _lib.load()
    for name in ("sgb_decoded_semantic_head", "sgb_decoded_semantic_head_workspace_bytes",
                 "sgb_decoded_feature_logits"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert len(lib.sgb_decoded_semantic_head.argtypes) == 13
    assert len(lib.sgb_decoded_feature_logits.argtypes) == 12


@pytest.mark.parametrize("kw,msg", [
    (dict(C=0), b"C = 0 outside [1, 1024]"),
    (dict(C=1025), b"C = 1025 outside [1, 1024]"),
    (dict(c=0), b"c = 0 outside [1, 128]"),
    (dict(c=129), b"c = 129 outside [1, 128]"),
    (dict(K=0), b"K = 0 outside [1, 1024]"),
    (dict(K=1025), b"K = 1025 outside [1, 1024]"),
    (dict(N=-1), b"N = -1 is negative"),
    (dict(first_class=-1), b"first_class = -1 outside [0, K = 5)"),
    (dict(first_class=5), b"first_class = 5 outside [0, K = 5)"),
    (dict(first_class=5, N=0), b"first_class = 5 outside [0, K = 5)"),
    (dict(render=None), b"null render"),
    (dict(weight=None), b"null weight"),
    (dict(text=None), b"null text"),
    (dict(ws=None), b"null workspace"),
    (dict(ws=264), b"workspace is not 16-byte aligned"),
    (dict(label=12), b"label is not 8-byte aligned"),
    (dict(render=None, sim=None), b"null render"),
    (dict(render=None, label=None), b"null render"),
])
def test_head_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _head(lib, **kw) == -1
    assert msg in lib.sgb_last_error()


@pytest.mark.parametrize("kw,msg", [
    (dict(C=0), b"C = 0 outside [1, 1024]"),
    (dict(c=129), b"c = 129 outside [1, 128]"),
    (dict(K=0), b"K = 0 outside [1, 1024]"),
    (dict(K=2000, Kpad=2000), b"K = 2000 outside [1, 1024]"),
    (dict(P=-1), b"P = -1 is negative"),
    (dict(Kpad=4), b"Kpad = 4 is less than K = 5"),
    (dict(features=None), b"null features"),
    (dict(weight=None), b"null weight"),
    (dict(text=None), b"null text"),
    (dict(out=None), b"null out"),
    (dict(ws=None), b"null workspace"),
    (dict(ws=8), b"workspace is not 16-byte aligned"),
])
def test_logits_reject_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _logits(lib, **kw) == -1
    assert msg in lib.sgb_last_error()


def test_nothing_to_do_is_not_an_error():
    """N = 0, P = 0 or no output requested: SGB_OK with any pointers (nothing is read or enqueued)."""
    lib = _lib.load()
    assert _head(lib, N=0, render=None, weight=None, text=None, ws=None) == 0
    assert _head(lib, sim=None, label=None, render=None, ws=None) == 0
    assert _logits(lib, P=0, features=None, out=None, ws=None) == 0


def test_widest_arguments_pass_validation():
    """C = 1024, c = 128, K = 1024 (and the narrowest) are accepted: with no GPU the call then fails in CUDA."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_decoded_head_gpu.py")
    lib = _lib.load()
    for C, c, K in ((1, 1, 1), (1024, 128, 1024)):
        assert _head(lib, C=C, c=c, K=K, first_class=0) == -2
        assert _head(lib, C=C, c=c, K=K, first_class=0, sim=None) == -2
        assert _logits(lib, C=C, c=c, K=K, Kpad=K, bias=1) == -2


def test_workspace_size_depends_on_the_widths_only():
    lib = _lib.load()
    ws = lib.sgb_decoded_semantic_head_workspace_bytes
    assert ws(512, 64, 21) > 0 and ws(512, 64, 21) % 256 == 0
    assert ws(768, 128, 201) > ws(512, 64, 21)
    # A (K x c, twice), beta and the float64 Gram table: no term of image size
    assert ws(1024, 128, 1024) < 2 * 1024 * 128 * 4 + 1024 * 4 + 128 * 128 * 8 + 128 * 8 + 8 * 256
    for C, c, K in ((0, 4, 5), (1025, 4, 5), (8, 0, 5), (8, 129, 5), (8, 4, 0), (8, 4, 1025)):
        assert ws(C, c, K) == 0


def _args(r=(4, 6, 5), w=(8, 4), t=(5, 8), b=None, wdtype=torch.float32):
    return torch.rand(r), torch.rand(w).to(wdtype), torch.rand(t), (torch.rand(b) if b is not None else None)


@pytest.mark.parametrize("kw,kwcall,msg", [
    ({}, {}, "must be CUDA tensors"),
    (dict(b=(8,)), {}, "must be CUDA tensors"),
    (dict(r=(3, 6, 5)), {}, r"rendering must be \(c,H,W\) with c = 4"),
    (dict(r=(4, 30)), {}, r"rendering must be a \(c,H,W\) tensor"),
    (dict(w=(8, 4, 1)), {}, r"weight must be \(C,c\)"),
    (dict(t=(5, 7)), {}, r"weight must be \(C,c\)"),
    (dict(t=(5, 8, 1)), {}, r"weight must be \(C,c\)"),
    (dict(b=(7,)), {}, r"weight must be \(C,c\)"),
    (dict(wdtype=torch.float64), {}, "weight and bias must be float32"),
    (dict(wdtype=torch.float16), {}, "weight and bias must be float32"),
    (dict(w=(1025, 4), t=(5, 1025)), {}, "1 <= C <= 1024"),
    (dict(r=(129, 6, 5), w=(8, 129)), {}, "1 <= c <= 128"),
    (dict(t=(1025, 8)), {}, "1 <= K <= 1024"),
    ({}, dict(first_class=5), "first_class 5 out of range"),
    ({}, dict(first_class=-1), "first_class -1 out of range"),
])
def test_head_python_layer_rejects_bad_arguments(kw, kwcall, msg):
    from semantic_gaussians_b200.semantic import decoded_semantic_head
    r, w, t, b = _args(**kw)
    with pytest.raises(ValueError, match=msg):
        decoded_semantic_head(r, w, t, bias=b, **kwcall)


def test_head_python_layer_rejects_non_tensors_and_integer_inputs():
    from semantic_gaussians_b200.semantic import decoded_semantic_head
    r, w, t, _ = _args()
    with pytest.raises(ValueError, match="weight must be a tensor"):
        decoded_semantic_head(r, [[1.0] * 4] * 8, t)
    with pytest.raises(ValueError, match="text_features must be a tensor"):
        decoded_semantic_head(r, w, None)
    with pytest.raises(ValueError, match="rendering must be a floating-point tensor"):
        decoded_semantic_head(r.to(torch.int32), w, t)


@pytest.mark.parametrize("kw,kwcall,msg", [
    (dict(r=(6, 4)), {}, "must be CUDA tensors"),
    (dict(r=(6, 3)), {}, r"features must be \(P,c\) with c = 4"),
    (dict(r=(6, 4, 1)), {}, r"features must be a \(P,c\) tensor"),
    (dict(r=(6, 4), b=(9,)), {}, r"weight must be \(C,c\)"),
    (dict(r=(6, 4), wdtype=torch.float64), {}, "weight and bias must be float32"),
    (dict(r=(6, 4)), dict(pad_to=0), "pad_to must be >= 1"),
])
def test_logits_python_layer_rejects_bad_arguments(kw, kwcall, msg):
    from semantic_gaussians_b200.semantic import decoded_feature_logits
    f, w, t, b = _args(**kw)
    with pytest.raises(ValueError, match=msg):
        decoded_feature_logits(f, w, t, bias=b, **kwcall)


def _tool(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")      # no device, on any machine
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "time_decoded_semantic.py"), *args],
                          capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)


def test_timing_tool_help_exits_zero():
    p = _tool("--help")
    assert p.returncode == 0, p.stderr[-2000:]
    assert "usage:" in p.stdout


def test_timing_tool_refuses_to_run_without_a_gpu():
    p = _tool()
    assert p.returncode != 0
    assert p.stderr.strip().splitlines()[-1] == "time_decoded_semantic.py needs a GPU", p.stderr[-2000:]
