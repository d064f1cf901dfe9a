"""Segmentation metrics: the reference's ``utils/metric.py`` with the confusion matrix counted on the GPU.

The reference's evaluation (``eval_segmentation.py``) ends every view with a device-to-host copy of the label map
and a numpy ``bincount``.  ``ConfusionMatrix.add`` enqueues the counting on the current stream instead
(``sgb_confusion_accumulate``: one kernel, no synchronisation), and ``matrix()`` reads the summed matrix once after
the last view.  ``get_iou`` / ``evaluate_confusion`` then compute, print and log exactly what the reference's
functions do, except that the class names are passed in rather than chosen from a dataset string.

For a 3D evaluation against labelled points (scan vertices), ``nearest_points`` / ``transfer_labels`` carry the labels
of the Gaussians (or of the voxels of the 3D network) onto the points by an exact nearest-neighbour query on the GPU
(``sgb_nearest``), and ``ConfusionMatrix.add`` counts them as it counts label maps."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib

_PRED_CODES = {torch.int32: 1, torch.int64: 2}                   # SGB_LABEL_I32, SGB_LABEL_I64
_GT_CODES = {torch.uint8: 0, torch.int32: 1, torch.int64: 2}     # SGB_LABEL_U8, _I32, _I64


class ConfusionMatrix:
    """Confusion matrix of ``num_classes`` classes accumulated on ``device``.

    ``counts`` is the full ``(num_classes + 1, num_classes + 1)`` int64 tensor the kernel adds into (rows:
    prediction, columns: ground truth, column 0 included); a data-parallel caller may ``all_reduce`` it (SUM)
    before reading ``matrix()``."""

    def __init__(self, num_classes: int, device=None):
        self.num_classes = int(num_classes)
        dev = torch.device("cuda" if device is None else device)
        if dev.type != "cuda":
            raise ValueError("ConfusionMatrix counts on a CUDA device")
        self.device = dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())
        nb = self.num_classes + 1
        # one buffer, so that matrix() reads counts and the invalid-pair count with one copy: nb*nb counts, then the
        # kernel's uint32 invalid counter in the low half of the last int64 (little-endian; the high half stays 0).
        # The uint64 counts never reach 2**63, so int64 holds them unchanged.
        self._buf = torch.zeros(nb * nb + 1, dtype=torch.int64, device=self.device)
        self.counts = self._buf[: nb * nb].view(nb, nb)
        self._invalid = self._buf[nb * nb:]
        self._call(0, None, _PRED_CODES[torch.int64], None, _GT_CODES[torch.int64], 0)   # validates num_classes

    def _call(self, n, pred_ptr, pred_code, gt_ptr, gt_code, pred_offset):
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(_lib.load().sgb_confusion_accumulate(n, pred_ptr, pred_code, gt_ptr, gt_code, pred_offset,
                                                       self.num_classes, self.counts.data_ptr(),
                                                       self._invalid.data_ptr(), stream),
                   "sgb_confusion_accumulate")

    def add(self, pred: torch.Tensor, gt: torch.Tensor, pred_offset: int = 0) -> None:
        """Count the pairs ``(pred + pred_offset, gt)`` of one view or a stack of views.

        ``pred``: int32 / int64 label map (``label_argmax``, ``semantic_head``, ``torch.argmax``); the reference's
        ``label += 1`` is ``pred_offset=1``.  ``gt``: uint8 / int32 / int64 with as many elements.  Any shape;
        non-contiguous inputs are copied.  Enqueued on the current stream of the accumulator's device; never
        synchronises.  Pairs the reference would reject are counted apart and make ``matrix()`` raise."""
        for name, t, codes in (("pred", pred, _PRED_CODES), ("gt", gt, _GT_CODES)):
            if not isinstance(t, torch.Tensor) or t.device != self.device:
                raise ValueError(f"{name} must be a CUDA tensor on {self.device}")
            if t.dtype not in codes:
                raise ValueError(f"{name} dtype {t.dtype} not supported (need one of {sorted(map(str, codes))})")
        if pred.numel() != gt.numel():
            raise ValueError(f"pred has {pred.numel()} elements, gt {gt.numel()}")
        if not -2**31 <= int(pred_offset) < 2**31:
            raise ValueError("pred_offset must fit int32")
        if pred.numel() == 0:
            return
        p, g = pred.contiguous(), gt.contiguous()
        with torch.cuda.device(self.device):
            self._call(p.numel(), p.data_ptr(), _PRED_CODES[p.dtype], g.data_ptr(), _GT_CODES[g.dtype],
                       int(pred_offset))

    def matrix(self) -> np.ndarray:
        """The ``(num_classes + 1, num_classes)`` uint64 matrix the reference's summed ``confusion`` would be
        (column 0 dropped).  Waits once for the device, so adds enqueued on any of its streams are included.
        Raises ValueError if any added pair was one the reference rejects (it raises on that view)."""
        torch.cuda.synchronize(self.device)
        host = self._buf.cpu().numpy()
        invalid = int(host[-1])
        if invalid:
            raise ValueError(f"{invalid} (pred, gt) pairs outside the confusion matrix: a negative label, or "
                             f"pred * {self.num_classes + 1} + gt >= {(self.num_classes + 1) ** 2}")
        nb = self.num_classes + 1
        return host[:-1].reshape(nb, nb).astype(np.uint64)[:, 1:]

    def reset(self) -> None:
        """Zero the counts and the invalid-pair count (enqueued on the current stream)."""
        self._buf.zero_()


def confusion_matrix(pred_ids: torch.Tensor, gt_ids: torch.Tensor, num_classes: int) -> np.ndarray:
    """``utils/metric.py::confusion_matrix`` for CUDA tensors: ``(num_classes + 1, num_classes)`` uint64."""
    if tuple(pred_ids.shape) != tuple(gt_ids.shape):
        raise ValueError(f"shapes differ: {tuple(pred_ids.shape)} vs {tuple(gt_ids.shape)}")
    cm = ConfusionMatrix(num_classes, pred_ids.device)
    cm.add(pred_ids, gt_ids)
    return cm.matrix()


def nearest_points(query: torch.Tensor, ref: torch.Tensor, max_distance: Optional[float] = None):
    """Exact nearest row of ``ref`` for every row of ``query``: ``(index int64 (M,), dist2 float32 (M,))``.

    ``query`` (M,3) and ``ref`` (P,3) are float32 CUDA tensors on one device, in the same frame (for scan vertices
    against Gaussians: the Gaussians' world frame).  ``dist2[q] = (dx*dx + dy*dy) + dz*dz`` in fp32 without FMA,
    ``index[q]`` the row that minimises it, the smallest row on ties.  ``max_distance`` is in scene units; a row
    matches only when ``dist2 <= float32(max_distance) * float32(max_distance)`` (that product rounded to fp32), and
    ``None`` sets no limit.  A query with no match, or with a non-finite coordinate, gets index -1 and dist2 +inf; a
    reference row with a non-finite coordinate is never returned.  Enqueued on the current stream, no synchronisation
    (``sgb_nearest``)."""
    for name, t in (("query", query), ("ref", ref)):
        if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.ndim != 2
                or t.shape[1] != 3):
            raise ValueError(f"{name} must be a float32 (N, 3) CUDA tensor")
    if query.device != ref.device:
        raise ValueError(f"query is on {query.device}, ref on {ref.device}: they must be on one device")
    max_dist2 = float("inf")
    if max_distance is not None:
        d = np.float32(max_distance)
        if not d >= 0:
            raise ValueError(f"max_distance must be a non-negative number or None, got {max_distance}")
        with np.errstate(over="ignore"):
            max_dist2 = float(d * d)
    q, r = query.detach().contiguous(), ref.detach().contiguous()
    M, P = q.shape[0], r.shape[0]
    index = torch.empty(M, dtype=torch.int64, device=q.device)
    dist2 = torch.empty(M, dtype=torch.float32, device=q.device)
    if M == 0:
        return index, dist2
    with torch.cuda.device(q.device):
        stream = torch.cuda.current_stream(q.device).cuda_stream
        ctx = _lib.ctx_for(q.device.index, stream)
        _lib.check(_lib.load().sgb_nearest(ctx, P, r.data_ptr(), M, q.data_ptr(), max_dist2, index.data_ptr(),
                                           dist2.data_ptr(), stream), "sgb_nearest")
    return index, dist2


def transfer_labels(query: torch.Tensor, ref: torch.Tensor, ref_labels: torch.Tensor,
                    max_distance: Optional[float] = None, fill: int = -1) -> torch.Tensor:
    """Label of the nearest ``ref`` row for every ``query`` row, ``fill`` where ``nearest_points`` finds no match:
    ``(M,)`` int64 on the device, with no synchronisation.  ``ref_labels`` is an integer CUDA tensor of P labels.
    With ``fill=-1`` and ``ConfusionMatrix.add(pred, gt, pred_offset=1)`` an unmatched point lands in prediction row 0,
    which ``get_iou`` counts as a false negative of its class."""
    if (not isinstance(ref_labels, torch.Tensor) or not isinstance(ref, torch.Tensor)
            or ref_labels.device != ref.device or tuple(ref_labels.shape) != tuple(ref.shape[:1])
            or ref_labels.dtype.is_floating_point or ref_labels.dtype.is_complex or ref_labels.dtype == torch.bool):
        raise ValueError("ref_labels must be an integer tensor of one label per ref row, on ref's device")
    index, _ = nearest_points(query, ref, max_distance)
    if ref.shape[0] == 0:
        return torch.full_like(index, int(fill))
    labels = ref_labels.to(torch.int64).index_select(0, index.clamp_min(0))
    return torch.where(index >= 0, labels, torch.full_like(labels, int(fill)))


def get_iou(label_id: int, confusion: np.ndarray):
    """IoU of one class: ``(iou, tp, tp + fp + fn)``, or ``nan`` when the class never occurs (0/0)."""
    # row label_id + 1: predicted as the class, column label_id: labelled as the class; union = tp + fp + fn
    tp = np.longlong(confusion[label_id + 1, label_id])
    union = np.longlong(confusion[label_id + 1].sum()) + np.longlong(confusion[:, label_id].sum()) - tp
    if union == 0:
        return float("nan")
    return float(tp) / union, tp, union


def evaluate_confusion(confusion: np.ndarray, class_labels: Sequence[str], stdout: bool = False,
                       log_path: Optional[str] = "eval_result.log"):
    """Per-class IoU and accuracy over the classes whose ground-truth column is not empty, their means, the
    reference's printed table (``stdout=True``) and log lines (appended to ``log_path``; None writes no file).
    Returns the mean IoU.  ``class_labels[i]`` names column i of ``confusion``."""
    if stdout:
        print("evaluating", confusion.sum(), "points...")
    print("num_classes:", len(class_labels))

    gt_total = confusion.sum(axis=0)
    class_ious, class_accs = {}, {}
    mean_iou, mean_acc, count = 0, 0, 0
    for i, name in enumerate(class_labels):
        if gt_total[i] == 0:
            continue
        class_ious[name] = get_iou(i, confusion)
        class_accs[name] = class_ious[name][1] / gt_total[i]
        count += 1
        mean_iou += class_ious[name][0]
        mean_acc += class_accs[name]
    mean_iou /= count
    mean_acc /= count

    def rows(fmt, missing):
        return [fmt.format(name, *class_ious[name]) if name in class_ious else name + missing for name in class_labels]

    if stdout:
        print("classes          IoU")
        print("----------------------------")
        for line in rows("{0:<14s}: {1:>5.3f}   ({2:>6d}/{3:<6d})", " error!"):
            print(line)
        print("Mean IoU", mean_iou)
        print("Mean Acc", mean_acc)
    if log_path is not None:
        with open(log_path, "a") as fp:
            fp.write("classes,IoU\n")
            for line in rows("{0:<14s}: {1:>5.3f}  ({2:>6d}/{3:<6d})", ",error"):
                fp.write(line + "\n")
            fp.write("mean IoU,{}\n".format(mean_iou))
            fp.write("mean Acc,{}\n\n".format(mean_acc))
    return mean_iou
