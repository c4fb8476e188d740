"""CPU: FusedEvaluator's host-side metric arithmetic against sklearn, state additivity, key names, and construction checks."""
import numpy as np
import pytest
import torch

from deepdfa_b200 import _lib
from deepdfa_b200.evaluator import FusedEvaluator, metrics_from_state, TP, FP, TN, FN, SAMPLES, LOSS_W, WEIGHT

sk = pytest.importorskip("sklearn.metrics")

KEYS = ("loss", "Accuracy", "Precision", "Recall", "F1Score", "confusion", "num_samples")


def _state(y_true, y_pred, loss_w=0.0, weight=0.0):
    s = np.zeros(_lib.EVAL_STATE_WORDS)
    y_true, y_pred = np.asarray(y_true, bool), np.asarray(y_pred, bool)
    s[TP] = np.sum(y_true & y_pred)
    s[FP] = np.sum(~y_true & y_pred)
    s[TN] = np.sum(~y_true & ~y_pred)
    s[FN] = np.sum(y_true & ~y_pred)
    s[SAMPLES] = y_true.size
    s[LOSS_W], s[WEIGHT] = loss_w, weight
    return torch.from_numpy(s)


def _check(y_true, y_pred):
    m = metrics_from_state(_state(y_true, y_pred), "val_")
    y_true, y_pred = np.asarray(y_true, int), np.asarray(y_pred, int)
    assert abs(m["val_Accuracy"] - sk.accuracy_score(y_true, y_pred)) < 1e-12
    assert abs(m["val_Precision"] - sk.precision_score(y_true, y_pred, zero_division=0)) < 1e-12
    assert abs(m["val_Recall"] - sk.recall_score(y_true, y_pred, zero_division=0)) < 1e-12
    assert abs(m["val_F1Score"] - sk.f1_score(y_true, y_pred, zero_division=0)) < 1e-12
    assert m["val_confusion"] == sk.confusion_matrix(y_true, y_pred, labels=[0, 1]).tolist()
    assert m["val_num_samples"] == y_true.size


@pytest.mark.parametrize("seed", range(8))
def test_metrics_match_sklearn_on_random_samples(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 500))
    _check(rng.random(n) < rng.random(), rng.random(n) < rng.random())


@pytest.mark.parametrize("y_true,y_pred", [
    ([0, 0, 0, 0], [0, 0, 0, 0]),          # all negative: precision / recall / F1 have zero denominators
    ([1, 1, 1], [1, 1, 1]),                # all positive
    ([0, 0, 1], [1, 1, 1]),                # everything predicted positive
    ([1, 1, 0], [0, 0, 0]),                # nothing predicted positive
    ([0, 1], [1, 0]),                      # no true positive
])
def test_metrics_match_sklearn_edge_cases(y_true, y_pred):
    _check(y_true, y_pred)


def test_sum_of_states_gives_the_metrics_of_the_concatenated_samples():
    rng = np.random.default_rng(7)
    a_t, a_p = rng.random(300) < 0.3, rng.random(300) < 0.4
    b_t, b_p = rng.random(170) < 0.6, rng.random(170) < 0.5
    sa, sb = _state(a_t, a_p, 0.7 * 4, 4), _state(b_t, b_p, 0.2 * 3, 3)
    both = metrics_from_state(sa + sb, "test_")
    cat = metrics_from_state(_state(np.r_[a_t, b_t], np.r_[a_p, b_p], 0.7 * 4 + 0.2 * 3, 7), "test_")
    assert both == cat
    assert abs(both["test_loss"] - (0.7 * 4 + 0.2 * 3) / 7) < 1e-15


@pytest.mark.parametrize("prefix", ["val_", "test_", "train_", ""])
def test_key_names_per_prefix(prefix):
    m = FusedEvaluator.metrics_from_state(_state([1, 0], [1, 1], 1.0, 2.0), prefix)
    assert sorted(m) == sorted(prefix + k for k in KEYS)
    assert m[f"{prefix}loss"] == 0.5


def test_loss_without_weight_is_nan():
    assert np.isnan(metrics_from_state(_state([], []), "val_")["val_loss"])


class _FakeModule:
    """Stands in for a CUDA module: construction checks run before any device work."""

    def __init__(self, encoder_mode=False, label_style="graph", layers=2):
        from types import SimpleNamespace
        self.hparams = SimpleNamespace(encoder_mode=encoder_mode, label_style=label_style)
        self._num_layers = layers
        self.device = torch.device("cuda", 0)


def test_encoder_mode_is_rejected():
    with pytest.raises(ValueError, match="encoder_mode"):
        FusedEvaluator(_FakeModule(encoder_mode=True, layers=0))


def test_unsupported_label_style_is_rejected():
    with pytest.raises(ValueError, match="label_style"):
        FusedEvaluator(_FakeModule(label_style="dataflow_solution_in"))


def test_cpu_module_is_rejected():
    from deepdfa_b200 import FlowGNNGGNNModule
    m = FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, 32, 2, 2, concat_all_absdf=True)
    with pytest.raises(_lib.DdfaError, match="CUDA"):
        FusedEvaluator(m)


def test_state_layout_matches_the_header():
    text = _lib.HEADER.read_text()
    assert f"#define DDFA_EVAL_STATE_WORDS {_lib.EVAL_STATE_WORDS}" in text
