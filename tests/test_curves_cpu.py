"""CPU: the NumPy restatement of torchmetrics < 0.10's threshold curves (tests/curve_rule.py) against a hand-computed case and
against scikit-learn where the two rules agree, and the curve entry points' argument checks (no GPU needed)."""
import os
import sys

import numpy as np
import pytest
import torch

from deepdfa_b200 import _lib, evaluator

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import curve_rule as R  # noqa: E402

sklearn_metrics = pytest.importorskip("sklearn.metrics")

Y = [1, 0, 1, 0, 0, 1, 0, 0]
P = [.9, .8, .8, .3, .2, .7, .1, .1]


def test_hand_computed_case():
    """Sorted: .9(+) .8(-) .8(+) .7(+) .3 .2 .1 .1 (all -): tps 1 2 3 3 3 3, full recall first at .7, so three thresholds where
    sklearn keeps all six."""
    thr, tps, fps = R.clf_curve(P, Y)
    assert thr.tolist() == np.float32([.9, .8, .7, .3, .2, .1]).tolist()
    assert tps.tolist() == [1, 2, 3, 3, 3, 3] and fps.tolist() == [0, 1, 1, 2, 3, 5]
    precision, recall, t = R.pr_curve(P, Y)
    assert t.tolist() == np.float32([.7, .8, .9]).tolist()
    np.testing.assert_array_equal(precision, [.75, 2 / 3, 1, 1])
    np.testing.assert_array_equal(recall, [1, 2 / 3, 1 / 3, 0])
    assert R.average_precision(precision, recall) == pytest.approx(0.80556, abs=5e-6)
    fpr, tpr, rt = R.roc_curve(P, Y)
    assert rt[0] == np.float32(np.float32(.9) + np.float32(1)) and rt[1:].tolist() == thr.tolist()
    assert fpr[0] == 0 and tpr[0] == 0
    assert R.auroc(fpr, tpr) == pytest.approx(0.9, abs=1e-15)
    _, _, sk_t = sklearn_metrics.precision_recall_curve(Y, np.float32(P))
    assert len(sk_t) == 6 and sk_t[-3:].tolist() == t.tolist()


def cases():
    rng = np.random.default_rng(0)
    out = []
    for n, kind in ((50, "random"), (1000, "random"), (20_000, "random"), (1000, "ties"), (20_000, "ties"), (300, "few")):
        y = (rng.random(n) < 0.06).astype(np.float32)
        y[:2] = [1, 0]
        if kind == "random":
            p = rng.random(n).astype(np.float32)
        elif kind == "ties":
            p = (np.floor(rng.random(n) * 256) / 256).astype(np.float32)      # multiples of 2^-8: heavy ties
        else:
            p = rng.choice(np.float32([0, .25, .5, 1]), n)
        out.append((f"{kind}-{n}", p, y))
    return out


@pytest.mark.parametrize("name,p,y", cases(), ids=[c[0] for c in cases()])
def test_against_sklearn_where_the_rules_agree(name, p, y):
    precision, recall, thr = R.pr_curve(p, y)
    sp, sr, st = sklearn_metrics.precision_recall_curve(y, p)
    L = len(thr)
    # sklearn keeps every threshold: the restatement is its tail from the first threshold at full recall on
    assert len(st) >= L and st[-L:].tolist() == thr.tolist()
    np.testing.assert_allclose(precision, sp[-(L + 1):], rtol=1e-15)
    np.testing.assert_allclose(recall, sr[-(L + 1):], rtol=1e-15)
    assert np.all(sr[:len(sr) - L - 1] == 1.0)          # what sklearn keeps beyond the cut is at full recall
    ap = R.average_precision(precision, recall)
    assert ap == pytest.approx(sklearn_metrics.average_precision_score(y, p), rel=1e-12)
    fpr, tpr, _ = R.roc_curve(p, y)
    assert R.auroc(fpr, tpr) == pytest.approx(sklearn_metrics.roc_auc_score(y, p), rel=1e-12)
    sf, stp, _ = sklearn_metrics.roc_curve(y, p, drop_intermediate=False)
    np.testing.assert_allclose(fpr, sf, rtol=1e-15)
    np.testing.assert_allclose(tpr, stp, rtol=1e-15)


def test_binned_rule():
    bins = R.default_bins()
    assert bins.dtype == np.float32 and len(bins) == 100 and bins[0] == 0 and bins[-1] == 1
    p = np.float32([0, .5, .5, 1, .25])
    y = [1, 0, 1, 1, 0]
    prec, rec, t = R.binned(p, y, np.float32([0, .5, 1]))
    tp, fp = np.float64([3, 2, 1]), np.float64([2, 1, 0])
    np.testing.assert_array_equal(prec, np.append((tp + 1e-6) / (tp + fp + 1e-6), 1))
    np.testing.assert_array_equal(rec, np.append(tp / (3 + 1e-6), 0))


def test_entry_points_check_their_arguments_without_a_gpu():
    L = _lib.lib()
    assert L.call("ddfa_curve_workspace_bytes", 1) > 0
    assert L.call("ddfa_curve_workspace_bytes", 10 ** 7) > L.call("ddfa_curve_workspace_bytes", 10 ** 6)
    rc = L.raw("ddfa_curve_sort")(None, None, 0, None, None, None, None, None, 0, None)
    assert rc == -1 and "n=0" in L.last_error()
    rc = L.raw("ddfa_curve_sort")(256, 256, 10, 256, 256, 256, 256, 256, 16, None)
    assert rc == -1 and "workspace" in L.last_error()
    rc = L.raw("ddfa_curve_sort")(256, 256, 10, 256, 260, 256, 256, 256, 1 << 20, None)
    assert rc == -1 and "aligned" in L.last_error()
    rc = L.raw("ddfa_curve_metrics")(*([256] * 3), 10, None, 5, *([256] * 10), 256, 1 << 20, None)
    assert rc == -1 and "NULL" in L.last_error()


def test_binary_curves_refuses_host_tensors():
    p = torch.tensor(P, dtype=torch.float32)
    y = torch.tensor(Y, dtype=torch.float32)
    with pytest.raises(_lib.DdfaError, match="CUDA tensor"):
        evaluator.binary_curves(p, y)
