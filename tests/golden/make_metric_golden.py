"""Generates tests/golden/metric_golden.npz by running the REFERENCE's own utils/metric.py (imported from
/root/reference) on seeded synthetic label maps.  Run in the build container:

    python tests/golden/make_metric_golden.py

evaluate_confusion appends to ./eval_result.log, so the reference runs in a temporary working directory.  Its class
names come from the reference's dataset tables; here they are replaced by the synthetic names of class_names() (the
module globals evaluate_confusion reads), so the fixtures and the tests share names without holding the tables.

Inputs are regenerated from the seed by the tests (metric_inputs); only outputs are stored, per case:
  <case>_matrix          the summed (num_classes + 1, num_classes) uint64 confusion matrix
  <case>_iou/_tp/_denom  get_iou of every class (nan / -1 where the ground-truth column is empty and
                         evaluate_confusion skips the class)
  <case>_mean_iou        evaluate_confusion's return value
  <case>_stdout          what evaluate_confusion(stdout=True) printed
  <case>_log             what it appended to eval_result.log"""
import contextlib
import importlib
import io
import os
import sys
import tempfile

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))

# case -> (num_classes, dataset string of the reference, seed, views, (H, W), classes left out of the ground truth,
#          fraction of ground-truth pixels set to num_classes + 1 where the flat bin still fits)
CASES = {
    "c19": (19, "scannet20", 1, 1, (48, 64), (), 0.0),
    "c20": (20, "cocomap", 2, 1, (37, 53), (), 0.0),
    "c19_empty": (19, "scannet20", 3, 1, (40, 40), (2, 7, 18), 0.0),
    "c20_wrap": (20, "cocomap", 4, 1, (33, 45), (5,), 0.05),
    "c19_views": (19, "scannet20", 5, 4, (30, 41), (11,), 0.02),
}


def class_names(n):
    """Synthetic class names, some longer than the 14-character column of the printed table."""
    return [f"label{i:02d}" + "-long-name" * (i % 3) for i in range(n)]


def metric_inputs(case):
    """[(pred int64 = rendering[1:].argmax, i.e. before the reference's `label += 1`; gt int32)] per view."""
    nc, _, seed, views, (h, w), absent, wrap = CASES[case]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(views):
        # blocky maps, like rendered label maps: an 8x8 grid of constant cells, 60 % of them predicted right, then
        # 20 % of the pixels random
        cells = (h // 8 + 1, w // 8 + 1)
        pc = rng.integers(0, nc, cells)
        gc = np.where(rng.random(cells) < 0.6, pc + 1, rng.integers(0, nc + 1, cells))
        pred = np.kron(pc, np.ones((8, 8), np.int64))[:h, :w]
        gt = np.kron(gc, np.ones((8, 8), np.int64))[:h, :w]
        noise = rng.random((h, w)) < 0.2
        pred = np.where(noise, rng.integers(0, nc, (h, w)), pred).astype(np.int64)
        gt = np.where(noise, rng.integers(0, nc + 1, (h, w)), gt)
        for a in absent:                            # class a never labelled: its column stays empty
            gt[gt == a + 1] = 0
        # gt = num_classes + 1 lands in row pred + 2, column 0 (the reference's flat bincount); legal while
        # pred + 1 < num_classes
        wrap_px = (rng.random((h, w)) < wrap) & (pred + 1 < nc)
        gt[wrap_px] = nc + 1
        out.append((pred, gt.astype(np.int32)))
    return out


def import_reference_metric():
    sys.path.insert(0, REF)
    try:
        return importlib.import_module("utils.metric")
    finally:
        sys.path.remove(REF)


def main():
    metric = import_reference_metric()
    out = {}
    cwd = os.getcwd()
    for case, (nc, dataset, *_rest) in CASES.items():
        names = class_names(nc)
        metric.SCANNET20_CLASS_LABELS = tuple(names) if dataset == "scannet20" else metric.SCANNET20_CLASS_LABELS
        metric.COCOMAP_CLASS_LABELS = tuple(names) if dataset == "cocomap" else metric.COCOMAP_CLASS_LABELS
        confusion = np.zeros((nc + 1, nc), dtype=np.ulonglong)
        for pred, gt in metric_inputs(case):
            label = pred + 1                                       # eval_segmentation.py: label += 1
            confusion += metric.confusion_matrix(label.reshape(-1), gt.reshape(-1), nc)
        iou, tp, denom = np.full(nc, np.nan), np.full(nc, -1, np.int64), np.full(nc, -1, np.int64)
        for i in range(nc):
            if confusion.sum(axis=0)[i] != 0:
                iou[i], tp[i], denom[i] = metric.get_iou(i, confusion)
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                buf = io.StringIO()
                with contextlib.redirect_stdout(buf):
                    mean_iou = metric.evaluate_confusion(confusion, stdout=True, dataset=dataset)
                log = open("eval_result.log").read()
            finally:
                os.chdir(cwd)
        out[f"{case}_matrix"] = confusion
        out[f"{case}_iou"], out[f"{case}_tp"], out[f"{case}_denom"] = iou, tp, denom
        out[f"{case}_mean_iou"] = np.float64(mean_iou)
        out[f"{case}_stdout"] = np.array(buf.getvalue())
        out[f"{case}_log"] = np.array(log)
    path = os.path.join(HERE, "metric_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, sorted(out))


if __name__ == "__main__":
    main()
