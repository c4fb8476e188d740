"""Statement-level localisation without a GPU: the metric of FusedEvaluator(statements=...) against the reference's own
eval_statements_list (tests/golden/reference_statement_golden.pt, made by tests/golden/make_reference_statement_golden.py), the host
restatement of ddfa_stmt_metric's ranking rule against Python's stable sort, the C ABI constants, and the error of the
integrated-gradients rule on the fp64 oracle."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import statement_rule as R  # noqa: E402

from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200.evaluator import STATEMENT_MODES, statement_metrics_from_state  # noqa: E402
from oracle import ggnn_oracle as O  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_statement_golden.pt")


def _cases():
    return torch.load(GOLDEN)["cases"]


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_statement_metrics_match_the_reference_exactly(case):
    st = R.host_state(case["scores"].numpy(), case["vuln"].numpy(), case["batch_num_nodes"].numpy(), full=True)
    m = statement_metrics_from_state(st, "test_", node_style=True)
    for k in range(1, 11):
        if case["vo"] is None:                # the reference divides by zero: no vulnerable function
            assert math.isnan(m[f"test_stmt_top{k}"])
        else:
            assert m[f"test_stmt_top{k}"] == case["vo"][k], (k, m[f"test_stmt_top{k}"], case["vo"][k])
        if case["all"] is None:
            assert math.isnan(m[f"test_stmt_all_top{k}"])
        else:
            assert m[f"test_stmt_all_top{k}"] == case["all"][k], (k, m[f"test_stmt_all_top{k}"], case["all"][k])
    assert m["test_stmt_functions"] == case["batch_num_nodes"].numel()


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_ranking_rule_equals_the_stable_sort(case):
    s, v, bnn = case["scores"].numpy(), case["vuln"].numpy(), case["batch_num_nodes"].numpy()
    n0 = 0
    for (vul, rank, _, _), n in zip(R.ranks(s, v, bnn), bnn.tolist()):
        if vul:
            assert rank == R.rank_by_sort(s[n0:n0 + n], v[n0:n0 + n])
        n0 += n


def test_golden_covers_the_edge_cases():
    cases = {c["name"]: c for c in _cases()}
    bnn = torch.cat([c["batch_num_nodes"] for c in cases.values()])
    assert (bnn == 1).sum() >= 10 and ((bnn > 1) & (bnn < 10)).any() and (bnn >= 1000).any()
    s = torch.cat([c["scores"] for c in cases.values()])
    assert (s == 0.5).any() and (s == torch.nextafter(torch.tensor(0.5), torch.tensor(1.0))).any()
    assert cases["all_vulnerable"]["all"] is None and cases["no_vulnerable"]["vo"] is None
    # ties between a vulnerable and a non-vulnerable statement decide a rank somewhere
    ties = 0
    for c in cases.values():
        n0 = 0
        for n in c["batch_num_nodes"].tolist():
            sc, vu = c["scores"][n0:n0 + n], c["vuln"][n0:n0 + n]
            ties += int(any(((sc == sc[i]) & (vu == 0)).any() for i in range(n) if vu[i]))
            n0 += n
    assert ties >= 10


def test_graph_style_keys_and_nan_rule():
    st = np.zeros(R.WORDS)
    m = statement_metrics_from_state(st, "val_")
    assert set(m) == {f"val_stmt_top{k}" for k in range(1, 11)} | {"val_stmt_ifa", "val_stmt_vuln_functions", "val_stmt_functions"}
    assert all(math.isnan(m[f"val_stmt_top{k}"]) for k in range(1, 11)) and math.isnan(m["val_stmt_ifa"])
    st[R.FUNCTIONS], st[R.VULN], st[R.HIT1 + 2], st[R.RANK_SUM] = 5, 4, 3, 10
    m = statement_metrics_from_state(torch.tensor(st), "val_")
    assert m["val_stmt_top3"] == 0.75 and m["val_stmt_ifa"] == 2.5 and m["val_stmt_vuln_functions"] == 4


def test_abi_constants_match_the_header():
    h = open(_lib.HEADER).read()
    for name, val in (("DDFA_STMT_STATE_WORDS", _lib.STMT_STATE_WORDS), ("DDFA_STMT_MODE_VULN_ONLY", _lib.STMT_MODE_VULN_ONLY),
                      ("DDFA_STMT_MODE_FULL", _lib.STMT_MODE_FULL), ("DDFA_STMT_SCORE_ABS", _lib.STMT_SCORE_ABS),
                      ("DDFA_STMT_SCORE_X_TIMES", _lib.STMT_SCORE_X_TIMES)):
        assert int(re.search(rf"#define {name} (\d+)", h).group(1)) == val
    assert R.WORDS == _lib.STMT_STATE_WORDS
    assert set(STATEMENT_MODES.values()) == {"graph", "node"}


def ig_completeness_error(m: int, seed: int = 0):
    """max_b |Σ_{n in b} IG_n - (logit_b(x) - logit_b(0))| of the rule at m steps, on the fp64 oracle."""
    feat = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
    torch.manual_seed(seed)
    o = O.OracleFlowGNNGGNN(feat, 1002, 32, 5, 3, concat_all_absdf=True).double()
    g = synth.make_batch(6, 40, seed=seed, variable=True, vuln_rate=0.5)
    ig = R.oracle_integrated_gradients(o, g, m)
    with torch.no_grad():
        x = o.embed(g)
        delta = R.oracle_logits_from_x(o, g, x) - R.oracle_logits_from_x(o, g, torch.zeros_like(x))
    bnn = g.batch_num_nodes()
    gid = torch.repeat_interleave(torch.arange(bnn.numel()), bnn)
    sums = torch.zeros(bnn.numel(), dtype=torch.float64).index_add_(0, gid, ig)
    return float((sums - delta).abs().max()), float(delta.abs().max())


# the completeness bound the GPU test applies to the device's integrated gradients at these m, relative to max |logit(x) - logit(0)|.
# The rule's own error depends on the batch and the weights (the MLP's ReLU kinks): 6.6e-4 at m = 50 on this small oracle batch,
# 3.5e-3 on the GPU test's C0 batch (H100, SIMT engine), hence the margin.
IG_COMPLETENESS_BOUND = {16: 2e-2, 50: 1e-2}


def test_integrated_gradients_completeness_on_the_oracle():
    e16, scale = ig_completeness_error(16)
    e50, _ = ig_completeness_error(50)
    e400, _ = ig_completeness_error(400)
    assert e16 <= IG_COMPLETENESS_BOUND[16] * max(scale, 1.0)
    assert e50 <= IG_COMPLETENESS_BOUND[50] * max(scale, 1.0)
    # more steps, smaller error (the MLP's ReLU kinks make the integrand non-smooth: slower than the midpoint rule's 1/m^2)
    assert e400 <= e50 / 2 and e50 <= e16
