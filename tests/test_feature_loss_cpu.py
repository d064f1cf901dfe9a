"""Feature-map distillation loss without a GPU: argument validation of sgb_feature_map_loss (every bad argument is
rejected before anything is enqueued) and the Python layer's ValueErrors."""
import pytest
import torch

from semantic_gaussians_b200 import _lib


def _call(lib, C=8, N=64, render=1, target=1, dtype=_lib.FEAT_F16, loss_type=_lib.FEATLOSS_COSINE, dL=1, loss=1):
    return lib.sgb_feature_map_loss(C, N, render, target, dtype, loss_type, dL, loss, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(C=0), b"C = 0 outside [1, 1024]"),
    (dict(C=-3), b"C = -3 outside [1, 1024]"),
    (dict(C=1025), b"C = 1025 outside [1, 1024]"),
    (dict(N=-1), b"N = -1 is negative"),
    (dict(dtype=2), b"unknown target_dtype 2"),
    (dict(dtype=-1), b"unknown target_dtype -1"),
    (dict(loss_type=3), b"unknown loss_type 3"),
    (dict(loss_type=-1), b"unknown loss_type -1"),
    (dict(loss=None), b"null loss"),
    (dict(loss=None, N=0), b"null loss"),
    (dict(render=None), b"null render"),
    (dict(target=None), b"null target"),
    (dict(dL=None), b"null dL_drender"),
])
def test_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _call(lib, **kw) == -1
    assert msg in lib.sgb_last_error()


def test_largest_width_passes_validation():
    """C = 1024 (and C = 1) are accepted: with no GPU the call then fails in CUDA, not in validation."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_feature_loss_gpu.py")
    lib = _lib.load()
    for C in (1, 1024):
        for lt in (_lib.FEATLOSS_COSINE, _lib.FEATLOSS_L1, _lib.FEATLOSS_L2):
            assert _call(lib, C=C, loss_type=lt, dtype=_lib.FEAT_F32) == -2


@pytest.mark.parametrize("render,target,kw,msg", [
    ((4, 6, 5), ((4, 6, 5), torch.float16), {}, "must be CUDA tensors"),
    ((4, 6, 5), ((4, 6, 5), torch.float32), {}, "must be CUDA tensors"),
    ((4, 6, 5), ((4, 6, 5), torch.float16), dict(loss_type="huber"), "loss_type must be one of"),
    ((4, 6, 5), ((4, 6, 6), torch.float16), {}, r"must both be \(C,H,W\)"),
    ((6, 5), ((6, 5), torch.float16), {}, r"must both be \(C,H,W\)"),
    ((4, 6, 5), ((4, 6, 5), torch.float64), {}, "target must be float16 or float32"),
    ((4, 6, 5), ((4, 6, 5), torch.bfloat16), {}, "target must be float16 or float32"),
    ((4, 6, 5), ((4, 6, 5), "grad"), {}, "target must not require grad"),
])
def test_python_layer_rejects_bad_arguments(render, target, kw, msg):
    from semantic_gaussians_b200.semantic import feature_map_loss_and_grad
    shape, dtype = target
    y = torch.rand(shape).requires_grad_(True) if dtype == "grad" else torch.rand(shape).to(dtype)
    with pytest.raises(ValueError, match=msg):
        feature_map_loss_and_grad(torch.rand(render), y, **kw)
