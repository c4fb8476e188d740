"""DeepLift, DeepLiftShap and GradientShap statement scores without a GPU: FusedEvaluator's argument checks, the three new
graph-style modes, known answers of the host draws that restate ddfa_stmt_shap_input (tests/attribution_rule.py), and hand cases of
the fp64 oracle's rescale rule."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attribution_rule as A  # noqa: E402
import statement_rule as R  # noqa: E402

from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200.evaluator import STATEMENT_MODES, FusedEvaluator  # noqa: E402
from oracle import ggnn_oracle as O  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


class _FakeModule:
    """Stands in for a CUDA module: the argument checks run before any device work."""

    def __init__(self, label_style="graph"):
        self.hparams = SimpleNamespace(encoder_mode=False, label_style=label_style)
        self._num_layers = 2
        self.device = torch.device("cuda", 0)


def test_the_three_modes_are_graph_style():
    new = {"deeplift", "deeplift_shap", "gradient_shap"}
    assert set(STATEMENT_MODES) == {"probability", "attention", "saliency", "integrated_gradients"} | new
    assert all(STATEMENT_MODES[k] == "graph" for k in new)


@pytest.mark.parametrize("mode", ["deeplift", "deeplift_shap", "gradient_shap"])
def test_node_style_is_rejected(mode):
    with pytest.raises(ValueError, match="label_style"):
        FusedEvaluator(_FakeModule("node"), statements=mode)


@pytest.mark.parametrize("kw,match", [
    (dict(statements="deeplift_shap", shap_samples=0), "shap_samples"),
    (dict(statements="gradient_shap", shap_samples=-3), "shap_samples"),
    (dict(statements="gradient_shap", baseline_stdev=-0.1), "baseline_stdev"),
    (dict(statements="gradient_shap", noise_stdev=-1.0), "noise_stdev"),
    (dict(statements="deeplift_shap", baseline_stdev=float("nan")), "baseline_stdev"),
    (dict(statements="gradient_shap", noise_stdev=float("inf")), "noise_stdev"),
    (dict(statements="deeplift", baseline_stdev=0.5), "baseline_stdev applies"),
    (dict(statements="deeplift_shap", noise_stdev=0.5), "noise_stdev applies"),
    (dict(statements="gradient_shap", attribution_seed=-1), "attribution_seed"),
    (dict(statements="gradient_shap", attribution_seed=2 ** 64), "attribution_seed"),
    (dict(statements="deeplift_shap", attribution_seed=1.5), "attribution_seed"),
    (dict(statements="gradient_shap", attribution_seed=True), "attribution_seed"),
])
def test_constructor_errors(kw, match):
    with pytest.raises(ValueError, match=match):
        FusedEvaluator(_FakeModule(), **kw)


def test_entry_points_are_declared():
    names = set(_lib.declared_symbols())
    assert {"ddfa_stmt_shap_input", "ddfa_stmt_attribution_score", "ddfa_mlp_dgrad_rescale"} <= names


# ---- the host draws -----------------------------------------------------------------------------------------------------------
def test_host_alpha_known_answers():
    # word 0 of Philox4x32-10(key 0, counter (0, 0, 0, ALPHA_WORD)) is 0xddb3d022: alpha = 0xddb3d0 / 2^24
    assert int(A._words(0, 0, 0, [0], A.ALPHA_WORD)[0][0]) == 0xddb3d022
    assert [int(v) for v in A.alphas(0, 0, 0, 4).astype(np.float64) * 2 ** 24] == [14529488, 4026780, 1756404, 8264737]
    assert [int(v) for v in A.alphas(7, 3, 2, 3).astype(np.float64) * 2 ** 24] == [2906373, 7168673, 11600342]
    a = A.alphas(7, 3, 2, 5000)
    assert a.dtype == np.float32 and a.min() >= 0 and a.max() < 1 and abs(float(a.mean()) - 0.5) < 0.02


def test_host_gaussian_known_answers():
    e = A.gaussians(0, 0, 0, 2, 8, False).reshape(-1)
    np.testing.assert_allclose(e[[0, 1, 2, 3, 8, 12]], [0.9911374751458971, -0.9246627803544332, -0.6176090549848544,
                                                        -0.4820683472644963, 1.067590023374167, -0.49077940114434454], rtol=1e-15)
    np.testing.assert_allclose(A.gaussians(5, 1, 3, 1, 4, True).reshape(-1),
                               [1.7251724261060493, 1.8286880397960183, 1.3153795275125924, 0.7437958728195656], rtol=1e-15)
    big = A.gaussians(11, 2, 0, 4000, 16, False)
    assert abs(big.mean()) < 0.01 and abs(big.std() - 1) < 0.01
    # the noise and the baseline of the same (batch, sample, node, column) are different draws, and so are the samples
    assert not np.allclose(A.gaussians(1, 0, 0, 3, 8, False), A.gaussians(1, 0, 0, 3, 8, True))
    assert not np.allclose(A.gaussians(1, 0, 0, 3, 8, False), A.gaussians(1, 0, 1, 3, 8, False))


# ---- the rescale rule on the oracle -------------------------------------------------------------------------------------------
def test_rescale_multiplier_hand_values():
    z = torch.tensor([2.0, -1.0, 3.0, -0.5, 1e-10], dtype=torch.float64)
    zr = torch.tensor([-1.0, -2.0, 1.0, 0.5, -1e-10], dtype=torch.float64)
    # (relu(z) - relu(z')) / (z - z'): 2/3; both dead: 0; both alive: 1; crossing downwards: (0 - 0.5) / -1 = 0.5; a step of 2e-10 (> eps): 1/2
    assert A.rescale_multiplier(z, zr).tolist() == [2.0 / 3.0, 0.0, 1.0, 0.5, 0.5]


def test_rescale_falls_back_to_the_derivative_below_eps():
    z = torch.tensor([0.5, -0.5, 1e-12, -1e-12], dtype=torch.float64)
    zr = z + 5e-11
    assert A.rescale_multiplier(z, zr).tolist() == [1.0, 0.0, 1.0, 0.0]
    # on the forward's side of the kink when it is given
    assert A.rescale_multiplier(z, zr, branch=torch.tensor([True, True, False, True])).tolist() == [1.0, 1.0, 0.0, 1.0]


def test_one_relu_head_by_hand():
    """Linear(2, 2) -> ReLU -> Linear(2, 1): d out / d pooled = W1 diag(m) W0 with the multipliers m worked out by hand."""
    lin0, lin1 = nn.Linear(2, 2).double(), nn.Linear(2, 1).double()
    with torch.no_grad():
        lin0.weight.copy_(torch.tensor([[1.0, 2.0], [-1.0, 1.0]]))
        lin0.bias.copy_(torch.tensor([0.5, -0.5]))
        lin1.weight.copy_(torch.tensor([[3.0, -2.0]]))
        lin1.bias.zero_()
    o = SimpleNamespace(output_layer=nn.Sequential(lin0, nn.ReLU(), lin1))
    p = torch.tensor([[1.0, 1.0]], dtype=torch.float64, requires_grad=True)
    ref = torch.tensor([[0.0, -1.0]], dtype=torch.float64)
    # z = (3.5, -0.5), z' = (-1.5, -1.5): m = (3.5 - 0) / 5 = 0.7 and (0 - 0) / 1 = 0
    A.head_rescaled(o, p, ref).sum().backward()
    assert torch.allclose(p.grad, torch.tensor([[3.0 * 0.7 * 1.0, 3.0 * 0.7 * 2.0]], dtype=torch.float64), rtol=0, atol=1e-15)


def _oracle(layers, seed=0):
    torch.manual_seed(seed)
    return O.OracleFlowGNNGGNN(FEAT, 1002, 8, 3, layers, concat_all_absdf=True).double()


def test_one_layer_deeplift_is_input_times_gradient():
    o = _oracle(1)
    g = synth.make_batch(5, 30, seed=1, variable=True, vuln_rate=0.5)
    with torch.no_grad():
        x = o.embed(g)
    dl = A.oracle_deeplift(o, g, [torch.zeros_like(x)])
    ixg = (x * R.oracle_input_grad(o, g, x)).sum(1)
    assert torch.allclose(dl, ixg, rtol=1e-12, atol=1e-14)


def test_deeplift_shap_of_zero_baselines_is_deeplift_and_the_head_rescale_matters():
    o = _oracle(3, seed=2)
    g = synth.make_batch(5, 30, seed=3, variable=True, vuln_rate=0.5)
    with torch.no_grad():
        x = o.embed(g)
    z = torch.zeros_like(x)
    dl = A.oracle_deeplift(o, g, [z])
    assert torch.allclose(A.oracle_deeplift(o, g, [z, z, z]), dl, rtol=1e-14, atol=0)
    ixg = (x * R.oracle_input_grad(o, g, x)).sum(1)
    assert not torch.allclose(dl, ixg, rtol=1e-6)


def test_gradient_shap_at_alpha_one_would_be_input_times_gradient():
    """GradientShap's per-sample term at α = 1 with a zero baseline is x · grad(x): the oracle's sample loop reaches it when
    the draws are replaced by 1."""
    o = _oracle(2, seed=4)
    g = synth.make_batch(4, 20, seed=5, variable=True, vuln_rate=0.5)
    with torch.no_grad():
        x = o.embed(g)
    orig = A.alphas
    try:
        A.alphas = lambda seed, batch, sample, n: np.ones(n, dtype=np.float32)
        gs = A.oracle_gradient_shap(o, g, 0, 0, 2)
    finally:
        A.alphas = orig
    assert torch.allclose(gs, (x * R.oracle_input_grad(o, g, x)).sum(1), rtol=1e-12, atol=1e-14)
