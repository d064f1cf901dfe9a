"""View-sharded multi-GPU execution (new in this framework; the reference is single-GPU).

The path shards by view: every rank holds a replica of the Gaussian tensors,
renders / fuses its own views, accumulates per-Gaussian sums locally in fp32 and then takes part in
ONE exchange step — a sum all-reduce of the (P, C) gradient or feature-sum tensor plus the small
geometry gradients / the view counts.  One process per GPU, torch.distributed for the plumbing
(NCCL over NVLink on the box, gloo in the CPU tests)."""
from __future__ import annotations

import os
from typing import Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist


def shard_range(n_items: int, rank: int, world: int) -> range:
    """Contiguous shard [r*V/G, (r+1)*V/G) of a view batch (K4: 32 views -> 4 per GPU on 8)."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    lo = (n_items * rank) // world
    hi = (n_items * (rank + 1)) // world
    return range(lo, hi)


def shard_strided(n_items: int, rank: int, world: int) -> range:
    """Strided shard r, r+G, ... (fusion: balances the per-view visibility across ranks)."""
    return range(rank, n_items, world)


def allreduce_sums(tensors: Sequence[torch.Tensor], group=None, bucket_bytes: int = 256 << 20) -> None:
    """In-place sum all-reduce of per-Gaussian accumulators.

    Large tensors go out in row-range buckets launched asynchronously back to back, so that the
    first buckets are already on the wire while later ones are still being enqueued and NCCL can
    pipeline them over NVLink; small tensors are flattened into one message.  No-op without an
    initialised process group or with world size 1."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    works = []
    small: List[torch.Tensor] = []
    for t in tensors:
        if t is None:
            continue
        if not t.is_contiguous():
            raise ValueError("allreduce_sums needs contiguous tensors (views are reduced in place)")
        nbytes = t.numel() * t.element_size()
        if nbytes <= (1 << 20):
            small.append(t)
            continue
        flat = t.view(-1)
        step = max(1, bucket_bytes // t.element_size())
        for s in range(0, flat.numel(), step):
            works.append(dist.all_reduce(flat[s:s + step], op=dist.ReduceOp.SUM, group=group, async_op=True))
    if small:
        buf = torch.cat([t.reshape(-1).to(torch.float32) for t in small])
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
        off = 0
        for t in small:
            n = t.numel()
            t.copy_(buf[off:off + n].view_as(t).to(t.dtype))
            off += n
    for w in works:
        w.wait()


def nccl_overlap_options():
    """Process-group options for ``dist.init_process_group("nccl", pg_options=...)``: NCCL's stream gets high
    priority.  The chain-backward kernel fills every SM for many waves; at equal priority the block
    scheduler keeps handing freed SM slots to ITS pending CTAs, so an all-reduce launched meanwhile only
    starts in the last wave.  With a high-priority stream the NCCL CTAs are placed as soon as the first
    chain CTAs retire."""
    opts = dist.ProcessGroupNCCL.Options()
    opts.is_high_priority_stream = True
    max_ctas = int(os.environ.get("SGB_NCCL_MAX_CTAS", "0"))
    if max_ctas > 0:  # fewer NCCL CTAs = fewer SMs taken from the overlapped chain-backward kernel
        opts.config.max_ctas = max_ctas
    return opts


class OverlappedFeatureGradReduce:
    """All-reduce of the (P, C) feature gradient overlapped with the rest of the backward pass.

    sgb_backward computes dL/dfeature FIRST and records a CUDA event when it is final
    (sgb_ctx_set_feature_grad_event, include/sgb200.h); the chain / geometry gradient kernels that follow
    only touch small tensors.  `start(grad)` — called right after `.backward()` returned on the host,
    while the GPU is still working through those kernels — makes a communication stream wait on that
    event only and launches the NCCL sum there; `finish()` joins it back into the current stream.

    The native event marks the moment the RAW gradient buffer is final.  That buffer is the leaf's ``.grad`` only
    when the leaf had no gradient before the backward (autograd then adopts the buffer); otherwise AccumulateGrad
    enqueues an in-place add AFTER the event and the early all-reduce would race with it.  `arm(param)` — called
    before `.backward()` — records which case applies; with a pre-existing ``.grad`` (a second local view,
    ``zero_grad(set_to_none=False)``) or without `arm`, `start` orders the exchange after everything enqueued on
    the current stream (correct, no overlap).
    Create the process group with ``nccl_overlap_options()`` or the overlap will not materialise."""

    def __init__(self, device: torch.device, group=None):
        from . import _lib
        self.device, self.group = torch.device(device), group
        with torch.cuda.device(self.device):
            self.comm_stream = torch.cuda.Stream(self.device, priority=-1)
            self.event = torch.cuda.Event()
            cur = torch.cuda.current_stream(self.device)
            self.event.record(cur)                      # materialises the cudaEvent_t
            self._ctx = _lib.ctx_for(self.device.index, cur.cuda_stream)
            _lib.set_feature_grad_event(self._ctx, self.event.cuda_event)
        self._work = None
        self._fresh = None          # None: unknown (arm() not called) -> conservative ordering

    def arm(self, param: torch.Tensor) -> None:
        """Call before ``.backward()``: remembers whether the leaf's gradient buffer will be adopted as is."""
        self._fresh = param.grad is None

    def start(self, feature_grad: torch.Tensor, fresh: Optional[bool] = None) -> None:
        if not feature_grad.is_contiguous():
            raise ValueError("feature gradient must be contiguous (reduced in place)")
        if fresh is None:
            fresh = bool(self._fresh)
        self._fresh = None
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.comm_stream):
            if fresh:
                self.comm_stream.wait_event(self.event)     # final right after the dL/dfeature kernel
            else:
                self.comm_stream.wait_stream(cur)           # an accumulate kernel follows the event: wait for it
            self._work = dist.all_reduce(feature_grad, op=dist.ReduceOp.SUM, group=self.group, async_op=True)

    def finish(self) -> None:
        if self._work is not None:
            self._work.wait()
            self._work = None
        torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)

    def close(self) -> None:
        from . import _lib
        self.finish()
        _lib.set_feature_grad_event(self._ctx, None)


def render_views_sharded(views: Sequence, render_fn, loss_fn, params: Iterable[torch.Tensor], group=None,
                         rank: Optional[int] = None, world: Optional[int] = None):
    """Forward + backward of this rank's shard of a view batch, gradients accumulated over the local
    views, then all-reduced: every rank ends with the same summed .grad on `params` as a single
    process rendering all views would have (up to fp32 re-association).

    render_fn(view) -> dict with "render"; loss_fn(view_index, render_dict) -> scalar tensor."""
    if rank is None:
        rank = dist.get_rank(group) if dist.is_initialized() else 0
    if world is None:
        world = dist.get_world_size(group) if dist.is_initialized() else 1
    params = [p for p in params]
    losses = []
    for i in shard_range(len(views), rank, world):
        out = render_fn(views[i])
        loss = loss_fn(i, out)
        loss.backward()                      # autograd accumulates into .grad across the local views
        losses.append(loss.detach())
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)     # a rank with an empty shard still joins the collective
    allreduce_sums([p.grad for p in params], group=group)
    total = torch.stack(losses).sum() if losses else torch.zeros((), device=params[0].device)
    if dist.is_initialized() and world > 1:
        dist.all_reduce(total, group=group)
    return total


def fuse_views_sharded(n_views: int, accumulate_view, feat_sum: torch.Tensor, count: torch.Tensor, normalize,
                       group=None, rank: Optional[int] = None, world: Optional[int] = None) -> None:
    """Fusion across ranks: rank r fuses views r, r+G, ... into its own (P,C) partial sum and count,
    one all-reduce merges them, then every rank normalises (fusion.py:146-147).

    accumulate_view(i) adds view i into feat_sum / count in place; normalize(feat_sum, count)."""
    if rank is None:
        rank = dist.get_rank(group) if dist.is_initialized() else 0
    if world is None:
        world = dist.get_world_size(group) if dist.is_initialized() else 1
    for i in shard_strided(n_views, rank, world):
        accumulate_view(i)
    allreduce_sums([feat_sum, count], group=group)
    normalize(feat_sum, count)
