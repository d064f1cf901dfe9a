"""Decoded feature-map loss without a GPU: the symbols are bound, sgb_decoded_feature_loss rejects every bad argument
before anything is enqueued, and the Python layer raises ValueError for bad tensors."""
import pytest
import torch

from semantic_gaussians_b200 import _lib


def _call(lib, C=8, c=4, N=64, render=1, weight=1, bias=None, target=1, dtype=_lib.FEAT_F16,
          loss_type=_lib.FEATLOSS_COSINE, dR=1, dW=1, db=None, ws=256, loss=1):
    return lib.sgb_decoded_feature_loss(C, c, N, render, weight, bias, target, dtype, loss_type, dR, dW, db, ws, loss,
                                        None)


def test_symbols_are_bound():
    lib = _lib.load()
    for name in ("sgb_decoded_feature_loss", "sgb_decoded_feature_loss_workspace_bytes"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert len(lib.sgb_decoded_feature_loss.argtypes) == 15


@pytest.mark.parametrize("kw,msg", [
    (dict(C=0), b"C = 0 outside [1, 1024]"),
    (dict(C=-3), b"C = -3 outside [1, 1024]"),
    (dict(C=1025), b"C = 1025 outside [1, 1024]"),
    (dict(c=0), b"c = 0 outside [1, 128]"),
    (dict(c=129), b"c = 129 outside [1, 128]"),
    (dict(N=-1), b"N = -1 is negative"),
    (dict(dtype=2), b"unknown target_dtype 2"),
    (dict(dtype=-1), b"unknown target_dtype -1"),
    (dict(loss_type=3), b"unknown loss_type 3"),
    (dict(loss_type=-1), b"unknown loss_type -1"),
    (dict(loss=None), b"null loss"),
    (dict(loss=None, N=0), b"null loss"),
    (dict(dW=None), b"null dL_dweight"),
    (dict(dW=None, N=0), b"null dL_dweight"),
    (dict(db=1), b"dL_dbias given without bias"),
    (dict(bias=1), b"bias given without dL_dbias"),
    (dict(render=None), b"null render"),
    (dict(weight=None), b"null weight"),
    (dict(target=None), b"null target"),
    (dict(dR=None), b"null dL_drender"),
    (dict(ws=None), b"null workspace"),
    (dict(ws=264), b"workspace is not 16-byte aligned"),
])
def test_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _call(lib, **kw) == -1
    assert msg in lib.sgb_last_error()


def test_workspace_size_depends_on_the_widths_only():
    lib = _lib.load()
    ws = lib.sgb_decoded_feature_loss_workspace_bytes
    assert ws(512, 64, 1) == ws(512, 64, 968 * 1296) > 0
    assert ws(768, 128, 10) > ws(512, 64, 10) and ws(768, 128, 10) % 256 == 0
    for C, c, N in ((0, 4, 1), (1025, 4, 1), (8, 0, 1), (8, 129, 1), (8, 4, -1)):
        assert ws(C, c, N) == 0


def test_widest_decoder_passes_validation():
    """C = 1024 with c = 128 (and C = c = 1) are accepted: with no GPU the call then fails in CUDA, not in validation."""
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_decoder_loss_gpu.py")
    lib = _lib.load()
    for C, c in ((1, 1), (1024, 128)):
        for lt in (_lib.FEATLOSS_COSINE, _lib.FEATLOSS_L1, _lib.FEATLOSS_L2):
            assert _call(lib, C=C, c=c, loss_type=lt, dtype=_lib.FEAT_F32, bias=1, db=1) == -2


def _args(r=(4, 6, 5), w=(8, 4), y=((8, 6, 5), torch.float16), b=None, wdtype=torch.float32):
    shape, dtype = y
    yt = torch.rand(shape).requires_grad_(True) if dtype == "grad" else torch.rand(shape).to(dtype)
    return torch.rand(r), torch.rand(w).to(wdtype), yt, (torch.rand(b) if b is not None else None)


@pytest.mark.parametrize("kw,kwcall,msg", [
    ({}, {}, "must be CUDA tensors"),
    (dict(b=(8,)), {}, "must be CUDA tensors"),
    (dict(y=((8, 6, 5), torch.float32)), {}, "must be CUDA tensors"),
    ({}, dict(loss_type="huber"), "loss_type must be one of"),
    (dict(y=((8, 6, 6), torch.float16)), {}, r"rendering must be \(c,H,W\)"),
    (dict(y=((7, 6, 5), torch.float16)), {}, r"rendering must be \(c,H,W\)"),
    (dict(w=(8, 3)), {}, r"rendering must be \(c,H,W\)"),
    (dict(w=(8, 4, 1)), {}, r"rendering must be \(c,H,W\)"),
    (dict(r=(6, 5), y=((8, 6), torch.float16)), {}, r"rendering must be \(c,H,W\)"),
    (dict(b=(7,)), {}, r"rendering must be \(c,H,W\)"),
    (dict(y=((8, 6, 5), torch.float64)), {}, "target must be float16 or float32"),
    (dict(y=((8, 6, 5), torch.bfloat16)), {}, "target must be float16 or float32"),
    (dict(y=((8, 6, 5), "grad")), {}, "target must not require grad"),
    (dict(wdtype=torch.float64), {}, "weight and bias must be float32"),
    (dict(w=(1025, 4), y=((1025, 6, 5), torch.float16)), {}, "1 <= C <= 1024"),
    (dict(r=(129, 6, 5), w=(8, 129)), {}, "1 <= c <= 128"),
])
def test_python_layer_rejects_bad_arguments(kw, kwcall, msg):
    from semantic_gaussians_b200.semantic import decoded_feature_map_loss_and_grads
    r, w, y, b = _args(**kw)
    with pytest.raises(ValueError, match=msg):
        decoded_feature_map_loss_and_grads(r, w, y, bias=b, **kwcall)


def test_python_layer_rejects_a_non_tensor_weight():
    from semantic_gaussians_b200.semantic import decoded_feature_map_loss_and_grads
    r, _, y, _ = _args()
    with pytest.raises(ValueError, match="weight must be a tensor"):
        decoded_feature_map_loss_and_grads(r, [[1.0] * 4] * 8, y)
