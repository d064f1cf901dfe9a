"""numpy restatements the segmentation-metric tests compare against.

reference_confusion   utils/metric.py::confusion_matrix as eval_segmentation.py calls it (np.bincount of the flat
                      index, reshaped, column 0 dropped); raises ValueError on the inputs the reference rejects.
confusion_full        the counting rule of sgb_confusion_accumulate: the full (nb, nb) uint64 histogram and the
                      number of pairs the reference rejects (negative label or flat bin past the end)."""
import numpy as np


def reference_confusion(pred_ids, gt_ids, num_classes):
    nb = num_classes + 1
    flat = pred_ids * nb + gt_ids
    return np.bincount(flat, minlength=nb ** 2).reshape((nb, nb)).astype(np.ulonglong)[:, 1:]


def confusion_full(pred, gt, num_classes, pred_offset=0):
    nb = num_classes + 1
    pr = pred.astype(np.int64).ravel() + pred_offset
    g = gt.astype(np.int64).ravel()
    inside = (pr >= 0) & (pr < nb) & (g >= 0)
    prc = np.where(inside, pr, 0)
    ok = inside & (g < nb * nb - prc * nb)
    full = np.bincount((prc * nb + np.where(ok, g, 0))[ok], minlength=nb * nb).astype(np.uint64).reshape(nb, nb)
    return full, int((~ok).sum())
