"""CPU: the split voxel feature loss (forward and gradient passes on an fp32 / fp16 / bf16 network output) without a
device.  Both entry points are exported and reject every bad argument before any CUDA call, and
semantic.voxel_feature_loss rejects bad inputs with ValueError."""
import pytest
import torch

from semantic_gaussians_b200 import _lib, semantic

F16, F32, BF16 = _lib.FEAT_F16, _lib.FEAT_F32, _lib.FEAT_BF16
OK = dict(M=100, F=1536, out=256, odt=BF16, mask=256, K=10, C=768, head=1, y=256, dt=F16, lt=0, ws=256, loss=256,
          dloss=256, grad=256)


def _forward(lib, **kw):
    a = {**OK, **kw}
    return lib.sgb_voxel_feature_loss_forward(a["M"], a["F"], a["out"], a["odt"], a["mask"], a["K"], a["C"], a["head"],
                                              a["y"], a["dt"], a["lt"], a["ws"], a["loss"], None)


def _backward(lib, **kw):
    a = {**OK, **kw}
    return lib.sgb_voxel_feature_loss_backward(a["M"], a["F"], a["out"], a["odt"], a["K"], a["C"], a["head"], a["y"],
                                               a["dt"], a["lt"], a["ws"], a["dloss"], a["grad"], None)


def test_symbols_are_bound():
    lib = _lib.load()
    for name in ("sgb_voxel_feature_loss_forward", "sgb_voxel_feature_loss_backward"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == 14


SHARED = [(dict(M=-1), b"M = -1"), (dict(M=2**31), b"M = 2147483648"), (dict(C=0), b"C = 0"),
          (dict(C=1025, F=4096, head=0), b"C = 1025"), (dict(head=2), b"does not fit"),
          (dict(head=-1), b"does not fit"), (dict(K=101), b"K = 101"), (dict(K=-1), b"K = -1"),
          (dict(dt=BF16), b"target_dtype 2"), (dict(dt=7), b"target_dtype 7"), (dict(lt=3), b"loss_type"),
          (dict(odt=3), b"output_dtype 3"), (dict(odt=-1), b"output_dtype -1"), (dict(y=None), b"null target"),
          (dict(ws=None), b"null workspace"), (dict(ws=264), b"16-byte"), (dict(out=None), b"null output"),
          (dict(out=257), b"output is not 2-byte aligned"),
          (dict(out=258, odt=F32), b"output is not 4-byte aligned")]


@pytest.mark.parametrize("kw,msg", SHARED + [(dict(loss=None), b"null loss"), (dict(mask=None), b"null output / mask")])
def test_forward_rejects_bad_arguments(kw, msg):
    lib = _lib.load()
    assert _forward(lib, **kw) == -1
    assert msg in lib.sgb_last_error(), lib.sgb_last_error()
    assert lib.sgb_last_error().startswith(b"sgb_voxel_feature_loss_forward: ")


@pytest.mark.parametrize("kw,msg", SHARED + [
    (dict(dloss=None), b"null dloss"), (dict(dloss=None, M=0, K=0), b"null dloss"),
    (dict(grad=None), b"null output / grad"), (dict(grad=255), b"grad is not 2-byte aligned"),
    (dict(grad=258, odt=F32), b"grad is not 4-byte aligned")])
def test_backward_rejects_bad_arguments(kw, msg):
    lib = _lib.load()
    assert _backward(lib, **kw) == -1
    assert msg in lib.sgb_last_error(), lib.sgb_last_error()
    assert lib.sgb_last_error().startswith(b"sgb_voxel_feature_loss_backward: ")


def test_fused_entry_point_still_rejects_a_bf16_target():
    lib = _lib.load()
    assert lib.sgb_voxel_feature_loss(10, 8, 16, 16, 10, 8, 0, 16, BF16, 0, 16, 16, 16, None) == -1
    assert b"target_dtype 2" in lib.sgb_last_error()


def _args(M=6, F=1536, K=4, out_dtype=torch.float16, gt_dtype=torch.float16, C=768):
    mask = torch.zeros(M, dtype=torch.bool)
    mask[:K] = True
    return torch.zeros(M, F, dtype=out_dtype), mask, torch.zeros(K, C, dtype=gt_dtype)


@pytest.mark.parametrize("change,kw,match", [
    (dict(), dict(), "CUDA tensor"),
    (dict(out_dtype=torch.float64), dict(), "float32, float16 or bfloat16"),
    (dict(out_dtype=torch.int32), dict(), "float32, float16 or bfloat16"),
    (dict(gt_dtype=torch.bfloat16), dict(), "features_gt must be float16 or float32"),
    (dict(), dict(head=2), "does not fit"),
    (dict(), dict(head=-1), "does not fit"),
    (dict(C=1025, F=2048), dict(channels=1025), "channels <= 1024"),
    (dict(), dict(channels=512), r"features_gt must be \(K, 512\)"),
    (dict(), dict(loss_type="huber"), "loss_type"),
    (dict(K=7), dict(), "more than the 6 rows"),
])
def test_python_entry_point_rejects_bad_inputs(change, kw, match):
    output, mask, gt = _args(**change)
    with pytest.raises(ValueError, match=match):
        semantic.voxel_feature_loss(output, mask, gt, **{"head": 1, **kw})


def test_python_entry_point_rejects_a_target_that_requires_grad():
    output, mask, gt = _args()
    with pytest.raises(ValueError, match="must not require grad"):
        semantic.voxel_feature_loss(output, mask, gt.float().requires_grad_(True), head=1)
