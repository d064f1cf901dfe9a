"""ctypes binding of libsgb200.so (include/sgb200.h).  The CUDA library is the product: if it is
missing or cannot be loaded, importing any rasterizer entry point raises — there is no fallback."""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsgb200.so")

SGB_OK = 0
DEPTH_NONE, DEPTH_F32, DEPTH_F64, DEPTH_SURFACE = 0, 1, 2, 3
FEAT_F16, FEAT_F32, FEAT_BF16 = 0, 1, 2
FEATLOSS_COSINE, FEATLOSS_L1, FEATLOSS_L2 = 0, 1, 2


class SgbError(RuntimeError):
    """Raised for any non-zero status of the native library (reference: std::runtime_error →
    RuntimeError through pybind, rasterizer_impl.cu:245, auxiliary.h:166-173)."""


class ViewInputs(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("D", C.c_int32), ("M", C.c_int32), ("W", C.c_int32), ("H", C.c_int32),
        ("C", C.c_int32),
        ("background", C.c_void_p), ("means3D", C.c_void_p), ("shs", C.c_void_p),
        ("colors_precomp", C.c_void_p), ("opacities", C.c_void_p), ("scales", C.c_void_p),
        ("scale_modifier", C.c_float),
        ("rotations", C.c_void_p), ("cov3D_precomp", C.c_void_p), ("viewmatrix", C.c_void_p),
        ("projmatrix", C.c_void_p), ("campos", C.c_void_p),
        ("tan_fovx", C.c_float), ("tan_fovy", C.c_float),
        ("prefiltered", C.c_int32), ("debug", C.c_int32), ("antialiasing", C.c_int32),
    ]


class ViewGrads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_dmeans3D", "dL_dcov3D",
        "dL_dsh", "dL_dscales", "dL_drotations")]


class Camera(C.Structure):
    """sgb_camera: the per-view fields of a batched call."""
    _fields_ = [("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float)]


class CameraGrads(C.Structure):
    """sgb_camera_grads: one view's camera-gradient outputs of an sgb_backward_*_cam call."""
    _fields_ = [("dL_dviewmatrix", C.c_void_p), ("dL_dprojmatrix", C.c_void_p), ("dL_dcampos", C.c_void_p)]


MAX_BATCH = 8


class FusionView(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("xyz", C.c_void_p), ("world_to_camera", C.c_void_p),
        ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
        ("w", C.c_int32), ("h", C.c_int32), ("cut_bound", C.c_int32), ("vis_thres", C.c_double),
        ("depth_mode", C.c_int32), ("depth", C.c_void_p),
    ]


ADAM_MAX_TENSORS = 8


class AdamTensor(C.Structure):
    """sgb_adam_tensor: one (rows, row_len) fp32 parameter table of an sgb_adam_step call."""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("visible", C.c_void_p), ("rows", C.c_int64), ("row_len", C.c_int32),
                ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("step_size", C.c_float), ("bias_correction2_sqrt", C.c_float)]


EXPORTS = (
    "sgb_last_error", "sgb_version", "sgb_ctx_create", "sgb_ctx_destroy", "sgb_ctx_scratch_bytes",
    "sgb_geometry_bytes", "sgb_binning_bytes", "sgb_image_bytes", "sgb_forward_geometry",
    "sgb_forward_render", "sgb_backward", "sgb_mark_visible", "sgb_state_field", "sgb_fusion_map",
    "sgb_fusion_accumulate", "sgb_fusion_normalize", "sgb_profile_enable", "sgb_profile_read",
    "sgb_profile_num_stages", "sgb_profile_stage_name", "sgb_ctx_launch_count",
    "sgb_ctx_set_feature_grad_event", "sgb_semantic_head", "sgb_feature_logits", "sgb_label_argmax", "sgb_ctx_view_stat", "sgb_knn_mean_dist2", "sgb_distill_loss",
    "sgb_forward_geometry_batch", "sgb_forward_render_batch", "sgb_backward_batch", "sgb_build_id",
    "sgb_photometric_forward", "sgb_photometric_backward", "sgb_confusion_accumulate", "sgb_feature_map_loss",
    "sgb_forward_render_batch_ext", "sgb_backward_batch_ext", "sgb_decoded_feature_loss",
    "sgb_decoded_feature_loss_workspace_bytes", "sgb_voxelize", "sgb_voxelize_workspace_bytes", "sgb_lift_batch",
    "sgb_adam_step", "sgb_coord_map_bytes", "sgb_coord_map_build", "sgb_coord_stride_workspace_bytes",
    "sgb_coord_stride", "sgb_kernel_map_workspace_bytes", "sgb_kernel_map_count", "sgb_kernel_map_fill",
    "sgb_sparse_conv_forward", "sgb_sparse_conv_backward_input", "sgb_sparse_conv_backward_weight_workspace_bytes",
    "sgb_sparse_conv_backward_weight", "sgb_voxelize_f64", "sgb_elastic_displace", "sgb_voxel_feature_loss",
    "sgb_voxel_feature_loss_workspace_bytes", "sgb_sparse_conv_half_forward_workspace_bytes",
    "sgb_sparse_conv_half_forward", "sgb_sparse_conv_half_backward_input_workspace_bytes",
    "sgb_sparse_conv_half_backward_input", "sgb_sparse_conv_half_backward_weight_workspace_bytes",
    "sgb_sparse_conv_half_backward_weight", "sgb_voxel_feature_loss_forward", "sgb_voxel_feature_loss_backward",
    "sgb_nearest", "sgb_decoded_semantic_head", "sgb_decoded_semantic_head_workspace_bytes",
    "sgb_decoded_feature_logits", "sgb_forward_render_joint_batch", "sgb_backward_joint_batch",
    "sgb_backward_batch_cam", "sgb_backward_joint_batch_cam",
)

_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """Load libsgb200.so once.  Raises ImportError (loudly) when the CUDA extension is absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: the sm_90a CUDA library is the rasterizer; build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
        lib.sgb_last_error.restype = C.c_char_p
        lib.sgb_version.restype = C.c_char_p
        lib.sgb_ctx_create.argtypes = [C.POINTER(vp), C.c_int]
        lib.sgb_ctx_destroy.argtypes = [vp]
        lib.sgb_ctx_destroy.restype = None
        lib.sgb_ctx_scratch_bytes.argtypes = [vp]
        lib.sgb_ctx_scratch_bytes.restype = C.c_size_t
        lib.sgb_geometry_bytes.argtypes = [i32]
        lib.sgb_geometry_bytes.restype = C.c_size_t
        lib.sgb_binning_bytes.argtypes = [i64]
        lib.sgb_binning_bytes.restype = C.c_size_t
        lib.sgb_image_bytes.argtypes = [i32, i32]
        lib.sgb_image_bytes.restype = C.c_size_t
        lib.sgb_forward_geometry.argtypes = [vp, C.POINTER(ViewInputs), vp, vp, C.POINTER(i64), vp]
        lib.sgb_forward_render.argtypes = [vp, C.POINTER(ViewInputs), i64, vp, vp, vp, vp, vp, vp, vp]
        lib.sgb_backward.argtypes = [vp, C.POINTER(ViewInputs), i64, vp, vp, vp, vp, vp,
                                     C.POINTER(ViewGrads), vp]
        pvp = C.POINTER(vp)
        lib.sgb_forward_geometry_batch.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera), pvp, pvp,
                                                   C.POINTER(i64), vp]
        lib.sgb_forward_render_batch.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera), C.POINTER(i64),
                                                 pvp, pvp, pvp, pvp, pvp, pvp, vp]
        lib.sgb_backward_batch.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera), C.POINTER(i64), pvp,
                                           pvp, pvp, pvp, pvp, C.POINTER(ViewGrads), vp]
        lib.sgb_forward_render_batch_ext.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera),
                                                     C.POINTER(i64), pvp, pvp, pvp, pvp, pvp, pvp, pvp, pvp, vp]
        lib.sgb_backward_batch_ext.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera), C.POINTER(i64),
                                               pvp, pvp, pvp, pvp, pvp, pvp, pvp, C.POINTER(ViewGrads), vp]
        lib.sgb_forward_render_joint_batch.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera),
                                                       C.POINTER(i64), pvp, pvp, pvp, pvp, pvp, pvp, pvp, pvp, vp,
                                                       i32, vp, pvp, vp]
        lib.sgb_backward_joint_batch.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera), C.POINTER(i64),
                                                 pvp, pvp, pvp, pvp, pvp, pvp, pvp, C.POINTER(ViewGrads), vp, i32, vp,
                                                 pvp, vp, vp]
        lib.sgb_backward_batch_cam.argtypes = lib.sgb_backward_batch_ext.argtypes[:-1] + [C.POINTER(CameraGrads), vp]
        lib.sgb_backward_joint_batch_cam.argtypes = (lib.sgb_backward_joint_batch.argtypes[:-1] +
                                                     [C.POINTER(CameraGrads), vp])
        lib.sgb_build_id.restype = C.c_char_p
        lib.sgb_mark_visible.argtypes = [i32, vp, vp, vp, vp, vp]
        lib.sgb_state_field.argtypes = [C.c_char_p, i32, i64, i32, i32, vp, vp, vp, vp, vp]
        lib.sgb_state_field.restype = i64
        lib.sgb_fusion_map.argtypes = [vp, C.POINTER(FusionView), vp, vp]
        lib.sgb_fusion_accumulate.argtypes = [vp, C.POINTER(FusionView), vp, i32, i32, vp, vp, vp, vp]
        lib.sgb_fusion_normalize.argtypes = [i32, i32, vp, vp, vp]
        lib.sgb_lift_batch.argtypes = [vp, C.POINTER(ViewInputs), i32, C.POINTER(Camera), pvp, i32, vp, vp, vp]
        lib.sgb_profile_enable.argtypes = [vp, C.c_int]
        lib.sgb_profile_read.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(i32)]
        lib.sgb_profile_stage_name.argtypes = [C.c_int]
        lib.sgb_profile_stage_name.restype = C.c_char_p
        lib.sgb_ctx_launch_count.argtypes = [vp, C.c_int]
        lib.sgb_ctx_launch_count.restype = C.c_uint64
        lib.sgb_ctx_set_feature_grad_event.argtypes = [vp, vp]
        lib.sgb_ctx_view_stat.argtypes = [vp, C.c_int]
        lib.sgb_knn_mean_dist2.argtypes = [vp, i32, vp, vp, vp]
        lib.sgb_nearest.argtypes = [vp, i64, vp, i64, vp, C.c_float, vp, vp, vp]
        lib.sgb_distill_loss.argtypes = [i32, i32, i64, vp, vp, vp, i32, vp, vp, vp]
        lib.sgb_ctx_view_stat.restype = i64
        lib.sgb_semantic_head.argtypes = [vp, i32, i32, i64, vp, vp, i32, vp, vp, vp]
        lib.sgb_feature_logits.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp]
        lib.sgb_label_argmax.argtypes = [i32, i32, i64, vp, vp, vp]
        lib.sgb_decoded_semantic_head.argtypes = [i32, i32, i32, i64, vp, vp, vp, vp, i32, vp, vp, vp, vp]
        lib.sgb_decoded_semantic_head_workspace_bytes.argtypes = [i32, i32, i32]
        lib.sgb_decoded_semantic_head_workspace_bytes.restype = C.c_size_t
        lib.sgb_decoded_feature_logits.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp]
        lib.sgb_photometric_forward.argtypes = [i32, i32, i32, vp, i64, i64, vp, i64, i64, vp, vp, vp]
        lib.sgb_photometric_backward.argtypes = [i32, i32, i32, vp, i64, i64, vp, i64, i64, vp, vp, vp, i64, i64, vp]
        lib.sgb_confusion_accumulate.argtypes = [i64, vp, i32, vp, i32, i32, i32, vp, vp, vp]
        lib.sgb_feature_map_loss.argtypes = [i32, i64, vp, vp, i32, i32, vp, vp, vp]
        lib.sgb_decoded_feature_loss.argtypes = [i32, i32, i64, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp]
        lib.sgb_decoded_feature_loss_workspace_bytes.argtypes = [i32, i32, i64]
        lib.sgb_decoded_feature_loss_workspace_bytes.restype = C.c_size_t
        lib.sgb_voxelize.argtypes = [i64, vp, C.POINTER(C.c_double), vp, vp, vp, vp, vp, vp]
        lib.sgb_voxelize_f64.argtypes = [i64, vp, C.POINTER(C.c_double), vp, vp, vp, vp, vp, vp]
        lib.sgb_voxelize_workspace_bytes.argtypes = [i64]
        lib.sgb_elastic_displace.argtypes = [i64, vp, i32, vp, i32, i32, i32, vp, C.c_double, vp, vp]
        lib.sgb_voxel_feature_loss_workspace_bytes.argtypes = [i64]
        lib.sgb_voxel_feature_loss_workspace_bytes.restype = C.c_size_t
        lib.sgb_voxel_feature_loss.argtypes = [i64, i32, vp, vp, i64, i32, i32, vp, i32, i32, vp, vp, vp, vp]
        lib.sgb_voxel_feature_loss_forward.argtypes = [i64, i32, vp, i32, vp, i64, i32, i32, vp, i32, i32, vp, vp, vp]
        lib.sgb_voxel_feature_loss_backward.argtypes = [i64, i32, vp, i32, i64, i32, i32, vp, i32, i32, vp, vp, vp, vp]
        lib.sgb_voxelize_workspace_bytes.restype = C.c_size_t
        lib.sgb_adam_step.argtypes = [C.POINTER(AdamTensor), i32, vp]
        pi64 = C.POINTER(i64)
        for name in ("sgb_coord_map_bytes", "sgb_coord_stride_workspace_bytes"):
            getattr(lib, name).argtypes = [i64]
            getattr(lib, name).restype = C.c_size_t
        lib.sgb_coord_map_build.argtypes = [i64, vp, vp, vp, vp]
        lib.sgb_coord_stride.argtypes = [i64, vp, i32, vp, vp, vp, vp]
        lib.sgb_kernel_map_workspace_bytes.argtypes = [i64, i32]
        lib.sgb_kernel_map_workspace_bytes.restype = C.c_size_t
        lib.sgb_kernel_map_count.argtypes = [i64, vp, vp, i64, vp, i32, i32, vp, vp, vp]
        lib.sgb_kernel_map_fill.argtypes = [i64, vp, vp, i64, vp, i32, i32, vp, vp, vp]
        lib.sgb_sparse_conv_forward.argtypes = [i32, pi64, vp, i32, i64, i32, vp, vp, i64, i32, vp, vp]
        lib.sgb_sparse_conv_backward_input.argtypes = [i32, pi64, vp, i32, i64, i32, vp, vp, i64, i32, vp, vp]
        lib.sgb_sparse_conv_backward_weight_workspace_bytes.argtypes = [i32, pi64, i32, i32]
        lib.sgb_sparse_conv_backward_weight_workspace_bytes.restype = C.c_size_t
        lib.sgb_sparse_conv_backward_weight.argtypes = [i32, pi64, vp, i32, i64, i32, vp, i64, i32, vp, vp, vp, vp]
        for name in ("sgb_sparse_conv_half_forward_workspace_bytes",
                     "sgb_sparse_conv_half_backward_input_workspace_bytes"):
            getattr(lib, name).argtypes = [i32, i32, pi64, i64, i32, i64, i32]
            getattr(lib, name).restype = C.c_size_t
        lib.sgb_sparse_conv_half_forward.argtypes = [i32, i32, pi64, vp, i32, i64, i32, vp, vp, i64, i32, vp, vp, vp]
        lib.sgb_sparse_conv_half_backward_input.argtypes = [i32, i32, pi64, vp, i32, i64, i32, vp, vp, i64, i32, vp, vp,
                                                            vp]
        lib.sgb_sparse_conv_half_backward_weight_workspace_bytes.argtypes = [i32, i32, pi64, i32, i32]
        lib.sgb_sparse_conv_half_backward_weight_workspace_bytes.restype = C.c_size_t
        lib.sgb_sparse_conv_half_backward_weight.argtypes = [i32, i32, pi64, vp, i32, i64, i32, vp, i64, i32, vp, vp,
                                                             vp, vp]
        _lib = lib
        return lib


def check(rc: int, what: str = "") -> None:
    if rc != SGB_OK:
        msg = load().sgb_last_error().decode("utf-8", "replace")
        raise SgbError(f"{what}: {msg} (status {rc})" if what else f"{msg} (status {rc})")


_ctxs = {}


def ctx_for(device_index: int, stream_handle: int) -> int:
    """One native scratch context per (device, stream): a ctx must not be shared by streams."""
    key = (device_index, stream_handle)
    h = _ctxs.get(key)
    if h is None:
        out = C.c_void_p()
        check(load().sgb_ctx_create(C.byref(out), device_index), "sgb_ctx_create")
        h = out.value
        _ctxs[key] = h
    return h


def profile_enable(ctx: int, on: bool = True) -> None:
    check(load().sgb_profile_enable(ctx, int(on)), "sgb_profile_enable")


def profile_read(ctx: int) -> dict:
    """{stage name: (summed ms, intervals)} since the previous read."""
    lib = load()
    n = lib.sgb_profile_num_stages()
    ms = (C.c_float * n)()
    cnt = (C.c_int32 * n)()
    check(lib.sgb_profile_read(ctx, ms, cnt), "sgb_profile_read")
    return {lib.sgb_profile_stage_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n)}


def set_feature_grad_event(ctx: int, cuda_event) -> None:
    """cuda_event: a cudaEvent_t handle (e.g. torch.cuda.Event.cuda_event after a first record) or None."""
    check(load().sgb_ctx_set_feature_grad_event(ctx, cuda_event), "sgb_ctx_set_feature_grad_event")


def view_stat(ctx: int, which: int) -> int:
    """0: blended (pixel, Gaussian) pairs of the last C > 4 view; 1: weight-row chunks in use."""
    return int(load().sgb_ctx_view_stat(ctx, which))


def build_id() -> str:
    """Identity string baked into the loaded library (version + hash of the sources it was built from)."""
    return load().sgb_build_id().decode()


def launch_count(ctx: int) -> tuple:
    lib = load()
    return int(lib.sgb_ctx_launch_count(ctx, 0)), int(lib.sgb_ctx_launch_count(ctx, 1))
