"""The C-ABI library loads without a GPU and exports every symbol include/sgb200.h declares;
argument validation (which runs before any CUDA call) reports the reference's messages."""
import ctypes as C
import os
import re

import pytest

from semantic_gaussians_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "sgb200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(sgb_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/sgb200.h but not exported"
    assert set(_lib.EXPORTS) <= set(names)
    assert b"sm_90a" in lib.sgb_version()


def test_library_contains_sm90a_code_with_bulk_and_tensor_copies():
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert "UBLKCP" in sass          # cp.async.bulk (TMA engine) staging of the per-tile Gaussian blocks
    assert "UTMALDG" in sass         # tensor-map tile copies of dfeature_persistent_kernel and chain_backward_warp_kernel


def test_state_sizes_are_sane():
    lib = _lib.load()
    assert lib.sgb_geometry_bytes(1_000_000) >= 1_000_000 * (32 + 24 + 12 + 3 + 4 + 4 + 4)
    assert lib.sgb_geometry_bytes(1_000_000) < 1_000_000 * 100          # reference: ~79 B / Gaussian + scan temp
    assert lib.sgb_binning_bytes(10_000_000) >= 40_000_000              # 4 B / instance (reference: 24 B + temp)
    assert lib.sgb_binning_bytes(10_000_000) < 41_000_000
    assert lib.sgb_image_bytes(1920, 1080) >= 1920 * 1080 * 8
    assert lib.sgb_geometry_bytes(0) > 0 and lib.sgb_binning_bytes(0) > 0


def _inputs(**kw):
    base = dict(P=10, D=0, M=0, W=64, H=64, C=3, background=1, means3D=1, shs=None, colors_precomp=1, opacities=1,
                scales=1, scale_modifier=1.0, rotations=1, cov3D_precomp=None, viewmatrix=1, projmatrix=1, campos=1,
                tan_fovx=0.5, tan_fovy=0.5, prefiltered=0, debug=0)
    base.update(kw)
    return _lib.ViewInputs(**base)


@pytest.mark.parametrize("kw,msg", [
    (dict(colors_precomp=None), b"excatly one of either SHs or precomputed colors"),
    (dict(shs=1, M=16, D=3), b"excatly one of either SHs or precomputed colors"),
    (dict(scales=None), b"scale/rotation pair or precomputed 3D covariance"),
    (dict(cov3D_precomp=1), b"scale/rotation pair or precomputed 3D covariance"),
    (dict(C=5, colors_precomp=None, shs=1, M=16, D=3), b"For non-RGB, provide precomputed Gaussian colors!"),
    (dict(W=0), b"invalid sizes"),
    (dict(colors_precomp=None, shs=1, M=4, D=3), b"SH degree 3 needs 16 coefficients"),
])
def test_argument_validation_happens_before_cuda(kw, msg):
    lib = _lib.load()
    inp = _inputs(**kw)
    R = C.c_int64(0)
    rc = lib.sgb_forward_geometry(None, C.byref(inp), None, None, C.byref(R), None)
    assert rc == -1
    assert msg in lib.sgb_last_error()


def test_ctx_create_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    out = C.c_void_p()
    rc = lib.sgb_ctx_create(C.byref(out), 0)
    assert rc == -2 and b"CUDA error" in lib.sgb_last_error()
    with pytest.raises(_lib.SgbError):
        _lib.check(rc, "sgb_ctx_create")


def test_missing_library_is_an_import_error(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "libsgb200.so"))
    with pytest.raises(ImportError, match="no CPU fallback"):
        _lib.load()


def test_shared_dcolors_with_sh_is_rejected_before_cuda():
    """With shs, every view of sgb_backward_batch needs its own dL_dcolors: the geometry kernel of view v reads it as
    view v's RGB gradient after view v's blend added into it.  A shared buffer is refused during argument checking
    (no ctx is dereferenced and no CUDA call is made, so this runs without a GPU)."""
    lib = _lib.load()
    V = 3
    inp = _inputs(colors_precomp=None, shs=1, M=16, D=3)
    cams = (_lib.Camera * V)(*[_lib.Camera(1, 1, 1, 0.5, 0.5) for _ in range(V)])
    arr = (C.c_void_p * V)(*[1] * V)
    R = (C.c_int64 * V)(*[1] * V)
    grads = (_lib.ViewGrads * V)(*[_lib.ViewGrads(*[1, 1, 1, 42, 1, 1, 1, 1, 1]) for _ in range(V)])
    rc = lib.sgb_backward_batch(1, C.byref(inp), V, cams, R, arr, arr, arr, arr, arr, grads, None)
    assert rc == -1
    assert b"dL_dcolors" in lib.sgb_last_error()
