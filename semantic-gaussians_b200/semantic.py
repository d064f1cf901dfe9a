"""Open-vocabulary semantic head on the GPU: what every ``render_chn`` caller of
the reference does with the rendered feature image (eval_segmentation.py:153-157, 253-257, 394-398;
view_viser.py:312-315) and with the per-Gaussian features (eval_segmentation.py:132, view_viser.py:185).

``semantic_head``      one pass over the (C,H,W) image: L2-normalise per pixel, similarities with the K
                       text embeddings, arg-max label map.
``feature_logits``     per-Gaussian similarities ``einsum("cq,dq->dc", text, features)``.
``render_semantic_labels``  label map WITHOUT the (C,H,W) feature image: alpha blending is linear in the
                       blended attribute, so rendering the K per-Gaussian similarities gives the same
                       un-normalised per-pixel similarities; the positive per-pixel normalisation does
                       not change the arg-max.
``distill_loss_and_grad``      training loss against per-pixel class labels and K class embeddings.
``feature_map_loss_and_grad``  training loss against a 2D model's feature map (cosine / l1 / l2).
``decoded_feature_map_loss_and_grads``  the same loss for a compact field through a per-pixel linear decoder.
``voxel_feature_loss_and_grad``  the same loss on the masked rows of a 3D network's (M, F) output (distill.py).
``voxel_feature_loss``  that loss as an autograd function of an fp32 / fp16 / bf16 output (mixed precision).
``decoded_semantic_head`` / ``decoded_feature_logits``  the head and the per-Gaussian logits of a compact field through
                       its linear decoder, without the decoded image or table."""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch.autograd.function import once_differentiable

from . import _lib


def _check(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (the semantic head has no CPU path)")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _stream_ctx(t: torch.Tensor):
    # callers hold `with torch.cuda.device(t.device)`: the kernels launch on a stream of t's device
    stream = torch.cuda.current_stream(t.device).cuda_stream
    return stream, _lib.ctx_for(t.device.index, stream)


def semantic_head(rendering: torch.Tensor, text_features: torch.Tensor, first_class: int = 1,
                  return_sim: bool = True, return_label: bool = True
                  ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """rendering (C,H,W), text_features (K,C)  ->  (sim (K,H,W) float32, label (H,W) int64) with

        r     = rendering / (rendering.norm(dim=0, keepdim=True) + 1e-8)
        sim   = torch.einsum("cq,qhw->chw", text_features, r)
        label = sim[first_class:].argmax(dim=0)          # the reference then adds 1 (class 0 = "other")
    """
    r = _check(rendering, "rendering")
    t = _check(text_features, "text_features").to(r.device)
    if r.ndim != 3 or t.ndim != 2 or t.shape[1] != r.shape[0]:
        raise ValueError("rendering must be (C,H,W) and text_features (K,C)")
    C_, H, W = r.shape
    K = t.shape[0]
    if not (0 <= first_class < K):
        raise ValueError("first_class out of range")
    sim = torch.empty((K, H, W), dtype=torch.float32, device=r.device) if return_sim else None
    label = torch.empty((H, W), dtype=torch.int64, device=r.device) if return_label else None
    with torch.cuda.device(r.device):
        stream, ctx = _stream_ctx(r)
        _lib.check(_lib.load().sgb_semantic_head(ctx, C_, K, H * W, r.data_ptr(), t.data_ptr(), first_class,
                                                sim.data_ptr() if sim is not None else None,
                                                label.data_ptr() if label is not None else None, stream),
                   "sgb_semantic_head")
    return sim, label


def feature_logits(features: torch.Tensor, text_features: torch.Tensor, pad_to: int = 1) -> torch.Tensor:
    """features (P,C), text_features (K,C) -> (P, Kpad) similarities, ``einsum("cq,dq->dc", text, features)``
    in columns [0,K), zeros in the padding columns (Kpad = K rounded up to a multiple of ``pad_to``)."""
    f = _check(features, "features")
    t = _check(text_features, "text_features").to(f.device)
    if f.ndim != 2 or t.ndim != 2 or t.shape[1] != f.shape[1]:
        raise ValueError("features must be (P,C) and text_features (K,C)")
    P, C_ = f.shape
    K = t.shape[0]
    Kpad = ((K + pad_to - 1) // pad_to) * pad_to
    out = torch.empty((P, Kpad), dtype=torch.float32, device=f.device)
    with torch.cuda.device(f.device):
        stream, _ = _stream_ctx(f)
        _lib.check(_lib.load().sgb_feature_logits(P, C_, K, Kpad, f.data_ptr(), t.data_ptr(), out.data_ptr(), stream),
                   "sgb_feature_logits")
    return out


def label_argmax(planes: torch.Tensor, num_classes: Optional[int] = None, first_class: int = 1) -> torch.Tensor:
    """planes (K',H,W) -> (H,W) int64 = planes[first_class:num_classes].argmax(dim=0)
    (``rendering[1:].argmax(dim=0)``, eval_segmentation.py:144)."""
    p = _check(planes, "planes")
    if p.ndim != 3:
        raise ValueError("planes must be (K,H,W)")
    K = p.shape[0] if num_classes is None else int(num_classes)
    if not (0 < K <= p.shape[0]) or not (0 <= first_class < K):
        raise ValueError("bad num_classes / first_class")
    H, W = p.shape[1:]
    label = torch.empty((H, W), dtype=torch.int64, device=p.device)
    with torch.cuda.device(p.device):
        stream, _ = _stream_ctx(p)
        _lib.check(_lib.load().sgb_label_argmax(K, first_class, H * W, p.data_ptr(), label.data_ptr(), stream),
                   "sgb_label_argmax")
    return label


def distill_loss_and_grad(rendering: torch.Tensor, class_emb: torch.Tensor, labels: torch.Tensor
                          ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Open-vocabulary distillation loss of a rendered (C,H,W) feature image against per-pixel class embeddings,
    and its gradient, in one pass over the image:

        loss = -(rendering * class_emb[labels].permute(2, 0, 1)).mean()          # labels (H,W) int32/int64
        grad = d loss / d rendering                                               # (C,H,W)

    Pixels whose label is outside [0, K) (ScanNet-style -1 / 255) are ignored: zero gradient, no loss term, and the
    mean runs over the valid pixels only.

    Returns (loss: 0-d float64 CUDA tensor, grad: (C,H,W) float32).  Use as ``rendering.backward(grad)``."""
    r = _check(rendering.detach(), "rendering")
    e = _check(class_emb, "class_emb").to(r.device)
    if r.ndim != 3 or e.ndim != 2 or e.shape[1] != r.shape[0]:
        raise ValueError("rendering must be (C,H,W) and class_emb (K,C)")
    if not labels.is_cuda or labels.dtype not in (torch.int32, torch.int64) or labels.numel() != r.shape[1] * r.shape[2]:
        raise ValueError("labels must be a CUDA int32/int64 tensor with H*W entries")
    lab = labels.contiguous()
    grad = torch.empty_like(r)
    loss2 = torch.zeros(2, dtype=torch.float64, device=r.device)      # [loss, number of non-ignored pixels]
    with torch.cuda.device(r.device):
        stream, _ = _stream_ctx(r)
        _lib.check(_lib.load().sgb_distill_loss(r.shape[0], e.shape[0], r.shape[1] * r.shape[2], r.data_ptr(),
                                               e.data_ptr(), lab.data_ptr(), int(lab.dtype == torch.int64),
                                               grad.data_ptr(), loss2.data_ptr(), stream), "sgb_distill_loss")
    return loss2[0], grad


_FEATURE_LOSSES = {"cosine": _lib.FEATLOSS_COSINE, "l1": _lib.FEATLOSS_L1, "l2": _lib.FEATLOSS_L2}
_FEATURE_MAX_C = 1024          # widest feature map the feature-loss kernels accept


def _feature_loss_codes(loss_type: str, target: torch.Tensor, name: str, grads_of: str) -> Tuple[int, int]:
    """(FEATLOSS_* code of loss_type, FEAT_* code of target's dtype) for the feature-loss entry points; ValueError
    for an unknown loss_type, a target that requires grad or one that is not float16 / float32."""
    if loss_type not in _FEATURE_LOSSES:
        raise ValueError(f"loss_type must be one of {sorted(_FEATURE_LOSSES)}, got {loss_type!r}")
    if target.requires_grad:
        raise ValueError(f"{name} must not require grad (the loss gives the gradient{grads_of} only)")
    if target.dtype not in (torch.float16, torch.float32):
        raise ValueError(f"{name} must be float16 or float32, got {target.dtype}")
    return _FEATURE_LOSSES[loss_type], _lib.FEAT_F16 if target.dtype == torch.float16 else _lib.FEAT_F32


def feature_map_loss_and_grad(rendering: torch.Tensor, target: torch.Tensor, loss_type: str = "cosine"
                              ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Distillation loss of a rendered (C,H,W) feature image against a 2D model's (C,H,W) feature map (fp16 or fp32,
    e.g. the OpenSeg / LSeg map ``fusion.fuse_scene`` consumes) and its gradient, in one pass over both images.
    With x = rendering.permute(1, 2, 0).reshape(-1, C) and y = target likewise (one row per pixel),
    the loss types of distill.py:111-124:

        "cosine"  m = y.norm(dim=-1) > 0;  (1 - torch.nn.CosineSimilarity()(x[m], y[m])).mean()   (0 if no m)
        "l1"      torch.nn.L1Loss()(x, y)
        "l2"      torch.nn.MSELoss()(x, y)

    Returns (loss: 0-d float64 CUDA tensor, grad: (C,H,W) float32 = d loss / d rendering).  Use as
    ``rendering.backward(grad)``.  Nothing is synchronised and no full-size temporary is allocated besides grad."""
    if not isinstance(rendering, torch.Tensor) or not isinstance(target, torch.Tensor):
        raise ValueError("rendering and target must be tensors")
    loss_code, dtype = _feature_loss_codes(loss_type, target, "target", " of the rendering")
    if rendering.ndim != 3 or target.shape != rendering.shape:
        raise ValueError(f"rendering and target must both be (C,H,W), got {tuple(rendering.shape)} and "
                         f"{tuple(target.shape)}")
    if not rendering.is_cuda or target.device != rendering.device:
        raise ValueError(f"rendering and target must be CUDA tensors on one device (the feature-map loss has no CPU "
                         f"path), got {rendering.device} and {target.device}")
    r = _check(rendering.detach(), "rendering")
    y = target.contiguous()
    C_, H, W = r.shape
    grad = torch.empty_like(r)
    loss2 = torch.empty(2, dtype=torch.float64, device=r.device)      # [loss, pixels averaged over]; zeroed by the call
    with torch.cuda.device(r.device):
        stream = torch.cuda.current_stream(r.device).cuda_stream
        _lib.check(_lib.load().sgb_feature_map_loss(C_, H * W, r.data_ptr(), y.data_ptr(), dtype, loss_code,
                                                   grad.data_ptr(), loss2.data_ptr(), stream), "sgb_feature_map_loss")
    return loss2[0], grad


def voxel_feature_loss_and_grad(output: torch.Tensor, mask: torch.Tensor, features_gt: torch.Tensor,
                                loss_type: str = "cosine", head: int = 0, channels: int = 768
                                ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The 3D distillation loss of distill.py:109-124 and its gradient, without gathering the masked rows.  With
    x = output[mask][:, head * channels : (head + 1) * channels] and y = features_gt.float():

        "cosine"  m = y.norm(dim=-1) > 0;  (1 - torch.nn.CosineSimilarity()(x[m], y[m])).mean()
        "l1"      torch.nn.L1Loss()(x, y)
        "l2"      torch.nn.MSELoss()(x, y)

    output: MinkUNet's (M, F) fp32 ``.F`` (read detached); mask: (M,) bool; features_gt: (mask.sum(), channels) fp16
    or fp32, one row per masked row in row order (``FeatureDataset`` / ``distill_targets`` give exactly that).

    Returns (loss, count, grad): 0-d float64 CUDA tensors and the (M, F) fp32 d loss / d output, zero outside the
    masked rows and the head's columns.  Use as ``out.F.backward(grad)``.  ``count`` is the number of rows averaged
    over (cosine: target rows with a non-zero element; l1 / l2: mask.sum()).  When it is 0 the loss and grad are 0;
    the reference ``continue``s past such a cosine batch (and l1 / l2 give NaN there), so a caller that wants the
    same skip reads ``count`` (one sync) and leaves out ``optimizer.step()``: a step with a zero gradient still
    applies AdamW's weight decay.  If mask.sum() is not features_gt's row count, loss and count are NaN.  Nothing
    is synchronised; every output is bitwise reproducible.  1 <= channels <= 1024, (head + 1) * channels <= F."""
    for name, t in (("output", output), ("mask", mask), ("features_gt", features_gt)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor (the voxel feature loss has no CPU path)")
    if not (output.device == mask.device == features_gt.device):
        raise ValueError("output, mask and features_gt must be on one device")
    if output.dtype != torch.float32 or output.ndim != 2:
        raise ValueError(f"output must be (M, F) float32, got {tuple(output.shape)} {output.dtype}")
    M, F = output.shape
    if mask.dtype != torch.bool or mask.shape != (M,):
        raise ValueError(f"mask must be ({M},) bool, got {tuple(mask.shape)} {mask.dtype}")
    loss_code, dtype = _feature_loss_codes(loss_type, features_gt, "features_gt", " of the output")
    if features_gt.ndim != 2 or features_gt.shape[1] != channels:
        raise ValueError(f"features_gt must be (K, {channels}) float16 or float32, got {tuple(features_gt.shape)} "
                         f"{features_gt.dtype}")
    if not 1 <= channels <= _FEATURE_MAX_C or head < 0 or (head + 1) * channels > F:
        raise ValueError(f"head {head} of {channels} channels does not fit in {F} columns "
                         f"(1 <= channels <= {_FEATURE_MAX_C})")
    if features_gt.shape[0] > M:
        raise ValueError(f"features_gt has {features_gt.shape[0]} rows, more than the {M} rows of output")
    x = output.detach().contiguous()
    y = features_gt.contiguous()
    m = mask.contiguous()
    grad = torch.empty_like(x)
    loss2 = torch.empty(2, dtype=torch.float64, device=x.device)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        nbytes = lib.sgb_voxel_feature_loss_workspace_bytes(M)
        if nbytes == 0:
            raise _lib.SgbError("sgb_voxel_feature_loss_workspace_bytes failed")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        _lib.check(lib.sgb_voxel_feature_loss(M, F, x.data_ptr(), m.data_ptr(), y.shape[0], channels, head,
                                              y.data_ptr(), dtype, loss_code, grad.data_ptr(), ws.data_ptr(),
                                              loss2.data_ptr(), stream), "sgb_voxel_feature_loss")
    return loss2[0], loss2[1], grad


_VOXEL_OUTPUT_DTYPES = {torch.float32: _lib.FEAT_F32, torch.float16: _lib.FEAT_F16, torch.bfloat16: _lib.FEAT_BF16}


class _VoxelFeatureLoss(torch.autograd.Function):
    """sgb_voxel_feature_loss_forward, and sgb_voxel_feature_loss_backward with the upstream gradient as dloss."""

    @staticmethod
    def forward(ctx, output, mask, features_gt, loss_code, target_code, head, channels):
        M, F = output.shape
        lib = _lib.load()
        nbytes = lib.sgb_voxel_feature_loss_workspace_bytes(M)
        if nbytes == 0:
            raise _lib.SgbError("sgb_voxel_feature_loss_workspace_bytes failed")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=output.device)
        loss2 = torch.empty(2, dtype=torch.float64, device=output.device)
        stream = torch.cuda.current_stream(output.device).cuda_stream
        _lib.check(lib.sgb_voxel_feature_loss_forward(M, F, output.data_ptr(), _VOXEL_OUTPUT_DTYPES[output.dtype],
                                                      mask.data_ptr(), features_gt.shape[0], channels, head,
                                                      features_gt.data_ptr(), target_code, loss_code, ws.data_ptr(),
                                                      loss2.data_ptr(), stream), "sgb_voxel_feature_loss_forward")
        # the workspace keeps the mask's row flags and ranks and the cosine count for the gradient pass
        ctx.save_for_backward(output, features_gt, ws)
        ctx.codes = (loss_code, target_code, head, channels)
        loss, count = loss2.unbind()
        ctx.mark_non_differentiable(count)
        return loss, count

    @staticmethod
    @once_differentiable
    def backward(ctx, dloss, _dcount):
        output, features_gt, ws = ctx.saved_tensors
        loss_code, target_code, head, channels = ctx.codes
        M, F = output.shape
        d = dloss.to(device=output.device, dtype=torch.float64).contiguous()
        grad = torch.empty_like(output)
        stream = torch.cuda.current_stream(output.device).cuda_stream
        _lib.check(_lib.load().sgb_voxel_feature_loss_backward(
            M, F, output.data_ptr(), _VOXEL_OUTPUT_DTYPES[output.dtype], features_gt.shape[0], channels, head,
            features_gt.data_ptr(), target_code, loss_code, ws.data_ptr(), d.data_ptr(), grad.data_ptr(), stream),
            "sgb_voxel_feature_loss_backward")
        return grad, None, None, None, None, None, None


def voxel_feature_loss(output: torch.Tensor, mask: torch.Tensor, features_gt: torch.Tensor,
                       loss_type: str = "cosine", head: int = 0, channels: int = 768
                       ) -> Tuple[torch.Tensor, torch.Tensor]:
    """``voxel_feature_loss_and_grad``'s loss as a differentiable function of the network output in its own dtype:
    MinkUNet's (M, F) ``.F`` in fp32, fp16 or bf16 (inside or outside autocast, ``output``'s dtype is used as given).
    The other arguments and their rules are ``voxel_feature_loss_and_grad``'s.

    Returns (loss, count), 0-d float64 CUDA tensors.  ``loss`` has a ``grad_fn``: ``loss.backward()``, or
    ``scaler.scale(loss).backward()`` with a ``torch.amp.GradScaler``, sends d loss / d output to ``output`` in
    output's dtype, computed as ``round(float(upstream) * g)`` with g the fp32 gradient ``voxel_feature_loss_and_grad``
    gives on ``output.float()``: the scale is applied before the one rounding, so a GradScaler scale keeps fp16
    gradients out of the subnormal range.  The loss and count are bitwise those of
    ``voxel_feature_loss_and_grad(output.float(), ...)``.  ``count`` is not differentiable.  Nothing is synchronised and
    nothing of output's size is allocated besides the gradient; output, features_gt and a workspace of about 9 bytes
    per row are kept for the backward pass.  Bitwise reproducible."""
    for name, t in (("output", output), ("mask", mask), ("features_gt", features_gt)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a tensor")
    if output.dtype not in _VOXEL_OUTPUT_DTYPES or output.ndim != 2:
        raise ValueError(f"output must be (M, F) float32, float16 or bfloat16, got {tuple(output.shape)} "
                         f"{output.dtype}")
    M, F = output.shape
    if mask.dtype != torch.bool or mask.shape != (M,):
        raise ValueError(f"mask must be ({M},) bool, got {tuple(mask.shape)} {mask.dtype}")
    loss_code, target_code = _feature_loss_codes(loss_type, features_gt, "features_gt", " of the output")
    if features_gt.ndim != 2 or features_gt.shape[1] != channels:
        raise ValueError(f"features_gt must be (K, {channels}) float16 or float32, got {tuple(features_gt.shape)} "
                         f"{features_gt.dtype}")
    if not 1 <= channels <= _FEATURE_MAX_C or head < 0 or (head + 1) * channels > F:
        raise ValueError(f"head {head} of {channels} channels does not fit in {F} columns "
                         f"(1 <= channels <= {_FEATURE_MAX_C})")
    if features_gt.shape[0] > M:
        raise ValueError(f"features_gt has {features_gt.shape[0]} rows, more than the {M} rows of output")
    for name, t in (("output", output), ("mask", mask), ("features_gt", features_gt)):
        if not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor (the voxel feature loss has no CPU path)")
    if not (output.device == mask.device == features_gt.device):
        raise ValueError("output, mask and features_gt must be on one device")
    with torch.cuda.device(output.device):
        return _VoxelFeatureLoss.apply(output.contiguous(), mask.contiguous(), features_gt.contiguous(), loss_code,
                                       target_code, int(head), int(channels))


def decoded_feature_map_loss_and_grads(rendering: torch.Tensor, weight: torch.Tensor, target: torch.Tensor,
                                       bias: Optional[torch.Tensor] = None, loss_type: str = "cosine"
                                       ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """``feature_map_loss_and_grad`` for a compact field: the rendered (c,H,W) image is lifted per pixel to the C
    channels of the (C,H,W) target (fp16 or fp32) by a linear decoder, ``x = weight @ r + bias`` (weight (C,c) as
    ``nn.Linear(c, C).weight``, or a 1x1 ``nn.Conv2d`` weight viewed as (C,c)), and the loss of
    ``feature_map_loss_and_grad`` is taken on x.  The decoded (C,H,W) image is never materialised.

    Returns (loss: 0-d float64 CUDA tensor, g_render (c,H,W), g_weight (C,c), g_bias (C,) or None when bias is None),
    all gradients of the loss.  Use as ``rendering.backward(g_render)``, ``decoder.weight.grad = g_weight``,
    ``decoder.bias.grad = g_bias``.  weight and bias are read detached (they may be nn.Parameters).  1 <= C <= 1024,
    1 <= c <= 128.  Nothing is synchronised; besides the outputs only a scratch buffer that depends on C and c alone
    is allocated, and every output is bitwise reproducible."""
    for name, t in (("rendering", rendering), ("weight", weight), ("target", target), ("bias", bias)):
        if not isinstance(t, torch.Tensor) and not (name == "bias" and t is None):
            raise ValueError(f"{name} must be a tensor")
    loss_code, dtype = _feature_loss_codes(loss_type, target, "target", "s of the rendering and decoder")
    if weight.dtype != torch.float32 or (bias is not None and bias.dtype != torch.float32):
        raise ValueError(f"weight and bias must be float32, got {weight.dtype} and "
                         f"{None if bias is None else bias.dtype}")
    if rendering.ndim != 3 or weight.ndim != 2 or weight.shape[1] != rendering.shape[0] or \
            target.shape != (weight.shape[0],) + tuple(rendering.shape[1:]) or \
            (bias is not None and tuple(bias.shape) != (weight.shape[0],)):
        raise ValueError(f"rendering must be (c,H,W), weight (C,c), target (C,H,W) and bias (C,), got "
                         f"{tuple(rendering.shape)}, {tuple(weight.shape)}, {tuple(target.shape)} and "
                         f"{None if bias is None else tuple(bias.shape)}")
    C_, c = weight.shape
    if not (1 <= C_ <= _FEATURE_MAX_C and 1 <= c <= 128):
        raise ValueError(f"the decoder must have 1 <= C <= {_FEATURE_MAX_C} outputs and 1 <= c <= 128 inputs, got "
                         f"({C_}, {c})")
    tensors = [rendering, weight, target] + ([bias] if bias is not None else [])
    if not rendering.is_cuda or any(t.device != rendering.device for t in tensors):
        raise ValueError(f"rendering, weight, target and bias must be CUDA tensors on one device (the decoded "
                         f"feature-map loss has no CPU path), got {', '.join(str(t.device) for t in tensors)}")
    r = _check(rendering.detach(), "rendering")
    w = weight.detach().contiguous()
    b = bias.detach().contiguous() if bias is not None else None
    y = target.contiguous()
    _, H, W = r.shape
    N = H * W
    lib = _lib.load()
    g_render = torch.empty_like(r)
    g_weight = torch.empty_like(w)
    g_bias = torch.empty_like(b) if b is not None else None
    workspace = torch.empty(lib.sgb_decoded_feature_loss_workspace_bytes(C_, c, N), dtype=torch.uint8, device=r.device)
    loss2 = torch.empty(2, dtype=torch.float64, device=r.device)      # [loss, pixels averaged over]; zeroed by the call
    with torch.cuda.device(r.device):
        stream = torch.cuda.current_stream(r.device).cuda_stream
        _lib.check(lib.sgb_decoded_feature_loss(C_, c, N, r.data_ptr(), w.data_ptr(),
                                                b.data_ptr() if b is not None else None, y.data_ptr(), dtype,
                                                loss_code, g_render.data_ptr(), g_weight.data_ptr(),
                                                g_bias.data_ptr() if g_bias is not None else None,
                                                workspace.data_ptr(), loss2.data_ptr(), stream),
                   "sgb_decoded_feature_loss")
    return loss2[0], g_render, g_weight, g_bias


_DECODED_MAX_K = 1024         # most classes the decoded head accepts


def _decoder_args(what: str, inputs, weight, text_features, bias, in_name: str, in_shape: str, c_dim: int,
                  first_class: int = 0) -> Tuple[torch.Tensor, ...]:
    """Checks shared by decoded_semantic_head and decoded_feature_logits: ``inputs`` (the c-channel rendering or
    features, of ``in_shape`` with c at ``c_dim``), weight (C,c), text_features (K,C), bias (C,) or None, all CUDA
    tensors on one device; weight and bias float32; 0 <= first_class < K.  Returns (inputs, weight, text, bias)
    detached, float32 and contiguous."""
    if not isinstance(inputs, torch.Tensor) or inputs.ndim != len(in_shape.split(",")):
        raise ValueError(f"{in_name} must be a ({in_shape}) tensor")
    for name, t in ((in_name, inputs), ("weight", weight), ("text_features", text_features), ("bias", bias)):
        if not isinstance(t, torch.Tensor) and not (name == "bias" and t is None):
            raise ValueError(f"{name} must be a tensor")
    if weight.dtype != torch.float32 or (bias is not None and bias.dtype != torch.float32):
        raise ValueError(f"weight and bias must be float32, got {weight.dtype} and "
                         f"{None if bias is None else bias.dtype}")
    for name, t in ((in_name, inputs), ("text_features", text_features)):
        if not t.is_floating_point():
            raise ValueError(f"{name} must be a floating-point tensor, got {t.dtype}")
    if weight.ndim != 2 or text_features.ndim != 2 or text_features.shape[1] != weight.shape[0] or \
            (bias is not None and tuple(bias.shape) != (weight.shape[0],)):
        raise ValueError(f"weight must be (C,c), text_features (K,C) and bias (C,), got {tuple(weight.shape)}, "
                         f"{tuple(text_features.shape)} and {None if bias is None else tuple(bias.shape)}")
    C_, c = weight.shape
    K = text_features.shape[0]
    if not (1 <= C_ <= _FEATURE_MAX_C and 1 <= c <= 128 and 1 <= K <= _DECODED_MAX_K):
        raise ValueError(f"the decoder must have 1 <= C <= {_FEATURE_MAX_C} outputs and 1 <= c <= 128 inputs, and "
                         f"1 <= K <= {_DECODED_MAX_K} classes, got (C, c) = ({C_}, {c}) and K = {K}")
    if inputs.shape[c_dim] != c:
        raise ValueError(f"{in_name} must be ({in_shape}) with c = {c} (weight's columns), got {tuple(inputs.shape)}")
    if not (0 <= first_class < K):
        raise ValueError(f"first_class {first_class} out of range for K = {K}")
    tensors = [inputs, weight, text_features] + ([bias] if bias is not None else [])
    if not inputs.is_cuda or any(t.device != inputs.device for t in tensors):
        raise ValueError(f"{in_name}, weight, text_features and bias must be CUDA tensors on one device (the {what} "
                         f"has no CPU path), got {', '.join(str(t.device) for t in tensors)}")
    return (inputs.detach().float().contiguous(), weight.detach().contiguous(),
            text_features.detach().float().contiguous(), bias.detach().contiguous() if bias is not None else None)


def decoded_semantic_head(rendering: torch.Tensor, weight: torch.Tensor, text_features: torch.Tensor,
                          bias: Optional[torch.Tensor] = None, first_class: int = 1, return_sim: bool = True,
                          return_label: bool = True) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """``semantic_head`` of a compact field's rendering through its linear decoder, without the decoded image:
    rendering (c,H,W), weight (C,c) (``nn.Linear(c, C).weight``), bias (C,) or None, text_features (K,C) ->
    (sim (K,H,W) float32 or None, label (H,W) int64 or None) with

        x     = torch.einsum("kc,chw->khw", weight, rendering) + bias[:, None, None]
        sim, label = semantic_head(x, text_features, first_class)

    The label is the arg-max of the un-normalised similarities (the positive per-pixel norm does not move it), so
    ``return_sim=False`` gives the same labels bitwise, reads the rendering once and never forms the norm.  ||x|| is a
    float64 quadratic form in the rendering, accurate where the decoded pixel is much shorter than its terms.  weight
    and bias are read detached (they may be nn.Parameters).  1 <= C <= 1024, 1 <= c <= 128, 1 <= K <= 1024.  Nothing
    is synchronised; besides the outputs only a scratch buffer that depends on C, c and K is allocated; bitwise
    reproducible."""
    r, w, t, b = _decoder_args("decoded semantic head", rendering, weight, text_features, bias, "rendering", "c,H,W", 0,
                               first_class)
    C_, c = w.shape
    K = t.shape[0]
    _, H, W = r.shape
    sim = torch.empty((K, H, W), dtype=torch.float32, device=r.device) if return_sim else None
    label = torch.empty((H, W), dtype=torch.int64, device=r.device) if return_label else None
    lib = _lib.load()
    with torch.cuda.device(r.device):
        ws = torch.empty(lib.sgb_decoded_semantic_head_workspace_bytes(C_, c, K), dtype=torch.uint8, device=r.device)
        stream = torch.cuda.current_stream(r.device).cuda_stream
        _lib.check(lib.sgb_decoded_semantic_head(C_, c, K, H * W, r.data_ptr(), w.data_ptr(),
                                                 b.data_ptr() if b is not None else None, t.data_ptr(), first_class,
                                                 sim.data_ptr() if sim is not None else None,
                                                 label.data_ptr() if label is not None else None, ws.data_ptr(),
                                                 stream), "sgb_decoded_semantic_head")
    return sim, label


def decoded_feature_logits(features: torch.Tensor, weight: torch.Tensor, text_features: torch.Tensor,
                           bias: Optional[torch.Tensor] = None, pad_to: int = 1) -> torch.Tensor:
    """``feature_logits`` of a compact field's (P,c) per-Gaussian features through its linear decoder: (P, Kpad) with
    ``einsum("cq,dq->dc", text, features @ weight.T + bias)`` in columns [0,K) and zeros in the padding columns
    (Kpad = K rounded up to a multiple of ``pad_to``), without forming the (P,C) decoded table.

    ``render_semantic_labels(..., logits=decoded_feature_logits(f, W, text, b, pad_to=4), bg_color=W @ bg_c + b)``
    renders the decoded label map straight from these: the blend weights and the final transmittance sum to one, so
    the constant text . b blends through unchanged as long as the background is decoded the same way."""
    if pad_to < 1:
        raise ValueError(f"pad_to must be >= 1, got {pad_to}")
    f, w, t, b = _decoder_args("decoded feature logits", features, weight, text_features, bias, "features", "P,c", 1)
    C_, c = w.shape
    P = f.shape[0]
    K = t.shape[0]
    Kpad = ((K + pad_to - 1) // pad_to) * pad_to
    out = torch.empty((P, Kpad), dtype=torch.float32, device=f.device)
    lib = _lib.load()
    with torch.cuda.device(f.device):
        ws = torch.empty(lib.sgb_decoded_semantic_head_workspace_bytes(C_, c, K), dtype=torch.uint8, device=f.device)
        stream = torch.cuda.current_stream(f.device).cuda_stream
        _lib.check(lib.sgb_decoded_feature_logits(P, C_, c, K, Kpad, f.data_ptr(), w.data_ptr(),
                                                  b.data_ptr() if b is not None else None, t.data_ptr(),
                                                  out.data_ptr(), ws.data_ptr(), stream), "sgb_decoded_feature_logits")
    return out


def render_semantic_labels(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, text_features: torch.Tensor,
                           features: Optional[torch.Tensor] = None, first_class: int = 1, scaling_modifier=1.0,
                           override_shape=None, foreground=None, world_rotate=None,
                           logits: Optional[torch.Tensor] = None) -> dict:
    """Label map of one view straight from per-Gaussian features, never writing the (C,H,W) image.

    Equivalent (up to fp32 re-association of the per-pixel sums) to the reference sequence
    ``render_chn(..., num_channels=C, override_color=features)`` -> normalise -> einsum -> ``sim[1:].argmax``:
    sum_c text[k][c] * (sum_j w_j f_j[c] + T bg[c]) = sum_j w_j (text[k].f_j) + T (text[k].bg).
    ``logits``: a precomputed ``feature_logits(features, text_features, pad_to=4)`` — it depends only on the
    scene and the label set, so an evaluation loop computes it once and passes it for every view.  For a compact
    field with a linear decoder, pass ``logits=decoded_feature_logits(f, W, text, b, pad_to=4)`` and the decoded
    background ``bg_color=W @ bg_c + b``: the blend weights and the final transmittance sum to one, so text . b
    blends through unchanged.
    Returns {"label": (H,W) int64, "logits": (K,H,W) un-normalised similarities, "radii", "visibility_filter"}."""
    from .renderer import render_chn
    t = _check(text_features, "text_features")
    K = t.shape[0]
    if logits is not None:
        g = _check(logits, "logits")
        if g.ndim != 2 or g.shape[1] < K or g.shape[1] % 4:
            raise ValueError("logits must be feature_logits(features, text_features, pad_to=4)")
    else:
        if features is None:
            features = pc._features_semantic
        g = feature_logits(features, t, pad_to=4)                  # (P, Kpad): 16-byte rows for the blend kernels
    bg = _check(bg_color, "bg_color").reshape(-1)
    bgk = torch.zeros(g.shape[1], dtype=torch.float32, device=g.device)
    bgk[:K] = t.to(g.device) @ bg.to(g.device)
    with torch.no_grad():
        out = render_chn(viewpoint_camera, pc, pipe, bgk, scaling_modifier=scaling_modifier, num_channels=g.shape[1],
                         override_color=g, override_shape=override_shape, foreground=foreground,
                         world_rotate=world_rotate)
    planes = out["render"]
    return {"label": label_argmax(planes, K, first_class), "logits": planes[:K], "radii": out["radii"],
            "visibility_filter": out["visibility_filter"]}
