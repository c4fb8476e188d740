"""CPU: the ranking rule of ddfa_predict_store against hand-written answers and against the kernel's key selection restated in
NumPy, the entry point's argument checks (reported before any launch), and FusedPredictor's construction checks."""
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import predict_rule as R  # noqa: E402

from deepdfa_b200 import _lib, build  # noqa: E402
from deepdfa_b200.predictor import FusedPredictor  # noqa: E402

INF, NAN = float("inf"), float("nan")


@pytest.mark.parametrize("scores,k,idx,top", [
    ([0.5, 0.9, 0.5, 0.5, 0.1], 3, [1, 0, 2], [0.9, 0.5, 0.5]),                 # a tie across the k boundary: node order decides
    ([0.5, 0.9, 0.5, 0.5, 0.1], 2, [1, 0], [0.9, 0.5]),
    ([-INF, 1.0, INF, -INF, INF], 5, [2, 4, 1, 0, 3], [INF, INF, 1.0, -INF, -INF]),
    ([NAN, -INF, NAN, 0.0, -0.0], 5, [3, 4, 1, 0, 2], [0.0, -0.0, -INF, NAN, NAN]),   # NaN after -inf, +0.0 ties -0.0
    ([NAN, NAN], 3, [0, 1, -1], [NAN, NAN, NAN]),
    ([], 3, [-1, -1, -1], [NAN, NAN, NAN]),                                      # an empty function
    ([2.0], 3, [0, -1, -1], [2.0, NAN, NAN]),
    ([1.0] * 40, 32, list(range(32)), [1.0] * 32),                               # all equal
])
def test_host_ranking_known_answers(scores, k, idx, top):
    i, s = R.top_k(scores, k)
    assert i.tolist() == idx
    assert R.same_floats(s, top)
    assert R.same_bits(s[np.array(idx) >= 0], np.asarray(top, np.float32)[np.array(idx) >= 0]), "raw scores: -0.0 stays -0.0"


@pytest.mark.parametrize("seed", range(6))
def test_key_selection_equals_the_stable_sort(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 300))
    s = (rng.integers(-3, 4, n) / 2).astype(np.float32)          # ties everywhere
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, np.float32(1e-45), -np.float32(1e-45)], np.float32)
    mask = rng.random(n) < 0.2
    s[mask] = rng.choice(special, int(mask.sum()))
    for k in (1, 10, 32):
        a_i, a_s = R.top_k(s, k)
        b_i, b_s = R.top_k_by_keys(s, k)
        assert np.array_equal(a_i, b_i) and R.same_floats(a_s, b_s)


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.lib()


def _call(L, **over):
    """ddfa_predict_store with valid graph-style arguments (fake pointers: a launch would fault) and ``over`` replaced."""
    a = dict(logits=256, node_probs=None, pooled=None, out_dim=0, scores=512, k=10, graph_ptr=768, num_graphs=4, num_valid=4,
             prob_out=1024, emb_out=None, top_idx=1280, top_score=1536, cursor=2048, capacity=100, stream=None)
    a.update(over)
    return L.raw("ddfa_predict_store")(*a.values())


@pytest.mark.parametrize("over,msg", [
    ({"k": 33}, "k=33"),
    ({"k": -1}, "k=-1"),
    ({"capacity": -1}, "capacity=-1"),
    ({"num_valid": 5}, "num_valid"),
    ({"node_probs": 4096}, "alternatives"),
    ({"prob_out": None}, "prob_out"),
    ({"logits": None}, "prob_out"),
    ({"emb_out": 4096}, "emb_out"),
    ({"pooled": 4096, "emb_out": 4096, "out_dim": 0}, "out_dim"),
    ({"scores": None}, "k > 0"),
    ({"top_idx": None}, "k > 0"),
    ({"k": 0}, "k > 0"),
    ({"cursor": None}, "cursor"),
    ({"cursor": 2052}, "8-byte"),
    ({"graph_ptr": None}, "graph_ptr"),
])
def test_argument_errors_are_reported_without_a_gpu(lib, over, msg):
    rc = _call(lib, **over)
    assert rc == -1 and msg in lib.last_error(), lib.last_error()


def test_no_function_is_a_no_op_without_a_gpu(lib):
    assert _call(lib, num_valid=0) == 0


class _FakeModule:
    """Stands in for a CUDA module: construction checks run before any device work."""

    def __init__(self, encoder_mode=False, label_style="graph", layers=2):
        from types import SimpleNamespace
        self.hparams = SimpleNamespace(encoder_mode=encoder_mode, label_style=label_style)
        self._num_layers = 0 if encoder_mode else layers
        self.device = torch.device("cuda", 0)


@pytest.mark.parametrize("kw,exc,msg", [
    ({"capacity": 0}, ValueError, "capacity"),
    ({"capacity": 2.5}, ValueError, "capacity"),
    ({"capacity": 10, "statements": "attention", "top_k": 33}, ValueError, "top_k"),
    ({"capacity": 10, "statements": "attention", "top_k": 0}, ValueError, "top_k"),
    ({"capacity": 10, "statements": "lime"}, ValueError, "statements"),
    ({"capacity": 10, "statements": "probability"}, ValueError, "label_style"),
    ({"capacity": 10, "statements": "saliency", "ig_steps": 0}, ValueError, "ig_steps"),
    ({"capacity": 10, "statements": "attention", "noise_stdev": 1.0}, ValueError, "noise_stdev"),
])
def test_graph_style_construction_checks(kw, exc, msg):
    with pytest.raises(exc, match=msg):
        FusedPredictor(_FakeModule(), **kw)


def test_node_style_takes_probability_only():
    with pytest.raises(ValueError, match="label_style"):
        FusedPredictor(_FakeModule(label_style="node"), 10, statements="attention")


def test_encoder_mode_takes_attention_only():
    for mode in ("saliency", "integrated_gradients", "deeplift", "gradient_shap"):
        with pytest.raises(ValueError, match="encoder_mode"):
            FusedPredictor(_FakeModule(encoder_mode=True), 10, statements=mode)
    with pytest.raises(ValueError, match="encoder_mode"):
        FusedPredictor(_FakeModule(encoder_mode=True, label_style="node"), 10)


def test_unsupported_label_style_and_cpu_module_are_rejected():
    with pytest.raises(ValueError, match="label_style"):
        FusedPredictor(_FakeModule(label_style="dataflow_solution_in"), 10)
    from deepdfa_b200 import FlowGNNGGNNModule
    m = FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, 32, 2, 2, concat_all_absdf=True)
    with pytest.raises(_lib.DdfaError, match="CUDA"):
        FusedPredictor(m, 10)


def test_max_k_matches_the_header():
    assert int(re.search(r"#define DDFA_PREDICT_MAX_K (\d+)", _lib.HEADER.read_text()).group(1)) == _lib.PREDICT_MAX_K
