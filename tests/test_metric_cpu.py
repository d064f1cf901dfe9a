"""CPU: segmentation metrics against fixtures of the reference's own utils/metric.py
(tests/golden/make_metric_golden.py), and argument validation of sgb_confusion_accumulate, which runs before any
CUDA call."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_metric_golden import CASES, class_names, metric_inputs  # noqa: E402
from metric_ref import confusion_full, reference_confusion  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402
from semantic_gaussians_b200.metric import evaluate_confusion, get_iou  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "metric_golden.npz"))


@pytest.mark.parametrize("case", sorted(CASES))
def test_counting_rule_matches_reference_matrix(case):
    """The kernel's counting rule (restated in numpy) gives the reference's summed matrix, wrap case included."""
    nc = CASES[case][0]
    total = np.zeros((nc + 1, nc + 1), np.uint64)
    for pred, gt in metric_inputs(case):
        full, invalid = confusion_full(pred, gt, nc, pred_offset=1)
        assert invalid == 0
        assert np.array_equal(full[:, 1:], reference_confusion(pred.reshape(-1) + 1, gt.reshape(-1), nc))
        total += full
    want = GOLDEN[f"{case}_matrix"]
    assert want.dtype == np.uint64 and np.array_equal(total[:, 1:], want)


def test_wrap_case_counts_in_the_next_row():
    full, invalid = confusion_full(np.array([3]), np.array([20]), 19)
    assert invalid == 0 and full[4, 0] == 1 and full.sum() == 1
    _, invalid = confusion_full(np.array([19]), np.array([20]), 19)     # flat bin == nb * nb: the reference raises
    assert invalid == 1


@pytest.mark.parametrize("case", sorted(CASES))
def test_get_iou_matches_reference(case):
    confusion = GOLDEN[f"{case}_matrix"]
    for i in range(CASES[case][0]):
        if GOLDEN[f"{case}_tp"][i] < 0:
            continue
        iou, tp, denom = get_iou(i, confusion)
        assert iou == GOLDEN[f"{case}_iou"][i] and tp == GOLDEN[f"{case}_tp"][i] and denom == GOLDEN[f"{case}_denom"][i]


def test_get_iou_of_an_absent_class_is_nan():
    confusion = np.zeros((4, 3), np.uint64)
    confusion[1, 0] = 5
    assert np.isnan(get_iou(2, confusion))


@pytest.mark.parametrize("case", sorted(CASES))
def test_evaluate_confusion_matches_reference(case, tmp_path, capsys):
    nc = CASES[case][0]
    log = tmp_path / "eval_result.log"
    log.write_text("earlier run\n")                                   # appended to, as the reference does
    mean_iou = evaluate_confusion(GOLDEN[f"{case}_matrix"], class_names(nc), stdout=True, log_path=str(log))
    assert mean_iou == GOLDEN[f"{case}_mean_iou"]
    assert capsys.readouterr().out == str(GOLDEN[f"{case}_stdout"])
    assert log.read_text() == "earlier run\n" + str(GOLDEN[f"{case}_log"])


def test_evaluate_confusion_quiet_and_without_log(tmp_path, monkeypatch, capsys):
    monkeypatch.chdir(tmp_path)
    case = "c19_empty"
    mean_iou = evaluate_confusion(GOLDEN[f"{case}_matrix"], class_names(19), log_path=None)
    assert mean_iou == GOLDEN[f"{case}_mean_iou"]
    assert capsys.readouterr().out == "num_classes: 19\n"              # printed even without stdout=True
    assert os.listdir(tmp_path) == []


def _counts():
    counts = (C.c_uint64 * 4)()
    invalid = C.c_uint32(0)
    return counts, invalid


@pytest.mark.parametrize("kw,msg", [
    (dict(N=-1), b"N = -1 < 0"),
    (dict(pred_dtype=0), b"pred dtype code 0"),
    (dict(pred_dtype=3), b"pred dtype code 3"),
    (dict(gt_dtype=-1), b"gt dtype code -1"),
    (dict(gt_dtype=3), b"gt dtype code 3"),
    (dict(num_classes=0), b"num_classes = 0"),
    (dict(num_classes=226), b"num_classes = 226"),
    (dict(counts=None), b"null counts"),
    (dict(invalid=None), b"null counts / invalid"),
    (dict(pred=None), b"null pred / gt"),
    (dict(gt=None), b"null pred / gt"),
])
def test_confusion_accumulate_argument_validation_happens_before_cuda(kw, msg):
    lib = _lib.load()
    counts, invalid = _counts()
    labels = (C.c_int64 * 4)()
    a = dict(N=4, pred=C.addressof(labels), pred_dtype=2, gt=C.addressof(labels), gt_dtype=2, pred_offset=0,
             num_classes=1, counts=C.addressof(counts), invalid=C.addressof(invalid))
    a.update(kw)
    rc = lib.sgb_confusion_accumulate(a["N"], a["pred"], a["pred_dtype"], a["gt"], a["gt_dtype"], a["pred_offset"],
                                      a["num_classes"], a["counts"], a["invalid"], None)
    assert rc == -1
    assert msg in lib.sgb_last_error()


@pytest.mark.parametrize("num_classes", [1, 200, 225])
def test_confusion_accumulate_with_no_pairs_launches_nothing(num_classes):
    """N == 0 returns before any CUDA call, so it succeeds here; ScanNet200 fits the per-CTA histogram."""
    lib = _lib.load()
    counts, invalid = _counts()
    rc = lib.sgb_confusion_accumulate(0, None, 1, None, 0, 1, num_classes, C.addressof(counts), C.addressof(invalid),
                                      None)
    assert rc == 0 and list(counts) == [0] * 4 and invalid.value == 0
