"""NumPy restatement of torchmetrics < 0.10's binary threshold curves, as BaseModule.test_epoch_end (base_module.py:348-383) runs
them over test_preds / test_labels (not a test module).  Shared by tests/test_curves_cpu.py, which checks it against a
hand-computed case and against scikit-learn, and tests/test_curves_gpu.py, which checks binary_curves against it.

- ``clf_curve``: ``_binary_clf_curve``: descending distinct thresholds (ties by value: ``preds[1:] - preds[:-1] == 0``, so -0.0
  ties +0.0 and is shown as +0.0 here) and the int64 counts tps / fps of samples with p >= threshold.
- ``pr_curve``: ``_precision_recall_curve_compute_single_class``: cut at the first index where tps reaches its last value,
  reversed, precision 1 / recall 0 appended.
- ``roc_curve``: ``_roc_compute_single_class``: a leading (0, 0) point at thresholds[0] + 1; fpr / tpr are 0 where their
  denominator is 0.
- ``binned``: ``BinnedPrecisionRecallCurve``: counts at p >= t, ``(TP + 1e-6) / (TP + FP + 1e-6)`` and ``TP / (TP + FN + 1e-6)``,
  then 1 / 0.
- ``average_precision``: ``-sum((r[1:] - r[:-1]) * p[:-1])`` over the PR curve; ``auroc``: the trapezoids of the ROC curve.

Ratios are fp64 from the exact counts (torchmetrics divides in the counts' float type); thresholds stay fp32.
"""
import numpy as np

EPS = 1e-6


def clf_curve(p, y):
    """(thresholds fp32 descending, tps int64, fps int64)."""
    p = np.asarray(p, np.float32).copy()
    p[p == 0] = 0.0
    pos = np.asarray(y) == 1
    order = np.argsort(-p, kind="stable")
    ps, ys = p[order], pos[order]
    ends = np.flatnonzero(np.append(ps[1:] != ps[:-1], True))
    tps = np.cumsum(ys, dtype=np.int64)[ends]
    return ps[ends], tps, ends.astype(np.int64) + 1 - tps


def pr_curve(p, y):
    thr, tps, fps = clf_curve(p, y)
    P = tps[-1]
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = tps / (tps + fps).astype(np.float64)
        recall = tps / np.float64(P)
    last = int(np.flatnonzero(tps == P)[0])
    sl = slice(0, last + 1)
    return np.append(precision[sl][::-1], 1.0), np.append(recall[sl][::-1], 0.0), thr[sl][::-1].copy()


def roc_curve(p, y):
    thr, tps, fps = clf_curve(p, y)
    tps, fps = np.append(0, tps), np.append(0, fps)
    thr = np.append(np.float32(thr[0] + np.float32(1)), thr).astype(np.float32)
    fpr = fps / np.float64(fps[-1]) if fps[-1] > 0 else np.zeros(len(thr))
    tpr = tps / np.float64(tps[-1]) if tps[-1] > 0 else np.zeros(len(thr))
    return fpr, tpr, thr


def binned(p, y, thresholds):
    p = np.asarray(p, np.float32)
    pos = np.asarray(y) == 1
    t = np.asarray(thresholds, np.float32)
    tp = np.array([np.count_nonzero(pos & (p >= ti)) for ti in t], np.float64)
    fp = np.array([np.count_nonzero(~pos & (p >= ti)) for ti in t], np.float64)
    fn = np.count_nonzero(pos) - tp
    return np.append((tp + EPS) / (tp + fp + EPS), 1.0), np.append(tp / (tp + fn + EPS), 0.0), t


def average_precision(precision, recall):
    return float(-np.sum((recall[1:] - recall[:-1]) * precision[:-1]))


def auroc(fpr, tpr):
    return float(np.sum((fpr[1:] - fpr[:-1]) * (tpr[:-1] + tpr[1:]) / 2.0))


def default_bins(k: int = 100):
    """BinnedPrecisionRecallCurve(thresholds=k)'s thresholds as recalled: torch.linspace(0, 1.0, k) in fp32."""
    import torch
    return torch.linspace(0, 1.0, k, dtype=torch.float32).numpy()
