"""CPU: what the fp32 oracle does at each non-finite injection site of tests/test_nonfinite_gpu.py — the facts those tests compare
the kernels against — and that the sites are what they claim to be (a one-node embedding row is used by exactly one node).

The reference decides in fp32 whether a step is finite, so the oracle runs in fp32 here; torch's ReLU passes NaN forward and
passes the gradient of a NaN activation backward, which is what the head kernels must do for the same non-finite sets."""
import math

import numpy as np
import pytest
import torch

from nonfinite_sites import (EMBED, GGNN, HEAD, INF, NAN, SITES, grad_flags, model_state, nonfinite, oracle_step, poison,
                             poison_batch, site_id, touched_rows)

HIDDEN = 32


@pytest.mark.parametrize("style", ["graph", "node"])
@pytest.mark.parametrize("B", [255, 256])
def test_poison_row_is_used_by_exactly_one_node(style, B):
    g, where = poison_batch(style, B)
    api = g.ndata["_ABS_DATAFLOW_api"]
    assert int((api == where["row"]).sum()) == 1 and int(api[where["node"]]) == where["row"]
    offs = where["offs"]
    assert offs[where["graph"]] <= where["node"] < offs[where["graph"] + 1]
    n_rows = g.batch_size if style == "graph" else g.num_nodes()
    assert n_rows == B                                   # B graphs, or B one-node rows of the node head
    assert offs[-1] == g.num_nodes() and len(offs) - 1 == g.batch_size


def _run(style, site, B=256, seed=3):
    g, where = poison_batch(style, B)
    sd = model_state(HIDDEN, style, seed)
    return g, where, oracle_step(poison(sd, site, where), g, style)


@pytest.mark.parametrize("style", ["graph", "node"])
@pytest.mark.parametrize("site", SITES, ids=site_id)
def test_every_site_reaches_the_logits_and_the_loss(style, site):
    if style == "node" and site[0].startswith("pooling."):
        pytest.skip("node style has no pooling")
    g, where, r = _run(style, site)
    bad = nonfinite(r["logits"])
    flags = grad_flags(r["grads"])
    print(f"{style} {site_id(site)}: {int(bad.sum())} / {bad.numel()} logits non-finite, loss {float(r['loss'])}, "
          f"non-finite grads {sorted(k for k, v in flags.items() if v)}")
    assert bad.any() and not math.isfinite(float(r["loss"]))
    # with the loss over every graph (node), a poisoned logit makes every parameter's gradient non-finite: the step is skipped
    assert all(flags.values()), sorted(k for k, v in flags.items() if not v)
    if site[0] == EMBED:
        # local poison: only the poisoned graph (graph style) or nodes of the poisoned graph (node style) go non-finite
        touched = torch.zeros_like(bad)
        touched[torch.from_numpy(touched_rows(where, style))] = True
        assert not (bad & ~touched).any()
        assert bool(bad[where["graph"] if style == "graph" else where["node"]])
        # the embedding tables: only rows used by the poisoned graph's nodes can get a non-finite gradient
        offs = where["offs"]
        for k, gr in r["grads"].items():
            if k.startswith("all_embeddings."):
                col = g.ndata["_ABS_DATAFLOW_" + k.split(".")[1]]
                rows = set(col[offs[where["graph"]]:offs[where["graph"] + 1]].tolist())
                bad_rows = set(torch.nonzero(nonfinite(gr).any(1)).flatten().tolist())
                assert bad_rows <= rows, k
        assert flags[EMBED]
    else:
        # a non-finite parameter element shared by every graph (node): every logit goes NaN
        assert bad.all(), site


@pytest.mark.parametrize("style", ["graph", "node"])
def test_hidden_bias_nan_makes_every_logit_loss_and_gradient_nan(style):
    """The case fmaxf(NaN, 0) = 0 in the head hides: torch's ReLU keeps NaN, so nothing stays finite."""
    _, _, r = _run(style, ("output_layer.0.bias", NAN))
    assert torch.isnan(r["logits"]).all() and math.isnan(float(r["loss"]))
    for k, gr in r["grads"].items():
        assert torch.isnan(gr).any(), k
    for k in HEAD[2:] + GGNN:         # output_layer.0's gradient is 0 in the rows of units no graph activates
        assert torch.isnan(r["grads"][k]).all(), k


def test_pooled_nan_gives_a_nan_logit_through_the_head():
    """A NaN pooled vector ends in a NaN logit in torch (it would be b_last + W_last . relu(b_0) with fmaxf's ReLU)."""
    _, where, r = _run("graph", (EMBED, NAN))
    assert torch.isnan(r["logits"][where["graph"]])
    assert int(nonfinite(r["logits"]).sum()) == 1


def test_torch_relu_passes_nan_forward_and_its_gradient_backward():
    """What the kernels' relu_nan and relu_grad restate: relu(NaN) = NaN, and threshold_backward drops the gradient where the
    activation is <= 0 only, so a NaN activation passes its gradient."""
    x = torch.tensor([NAN, -1.0, 0.0, -0.0, 2.0, INF, -INF], requires_grad=True)
    y = torch.relu(x)
    assert math.isnan(float(y[0])) and y[1:].detach().tolist() == [0.0, 0.0, 0.0, 2.0, INF, 0.0]
    y.backward(torch.full_like(x, 3.0))
    assert x.grad.tolist() == [3.0, 0.0, 0.0, 0.0, 3.0, 3.0, 0.0]
    # relu_grad(act, g) = act <= 0 ? 0 : g, act the ReLU's output
    act = y.detach()
    assert torch.equal(torch.where(act <= 0, torch.zeros_like(act), torch.full_like(act, 3.0)), x.grad)


@pytest.mark.parametrize("value", [NAN, INF, -INF])
def test_one_node_embedding_poison_is_local(value):
    """Graph style: one poisoned node makes exactly its graph's logit non-finite (NaN for every sign: the gate's dot product mixes
    +inf and -inf terms), and every other graph's logit equals the clean model's bit for bit."""
    g, where = poison_batch("graph", 256)
    sd = model_state(HIDDEN, "graph", 3)
    clean = oracle_step(sd, g, "graph")
    r = oracle_step(poison(sd, (EMBED, value), where), g, "graph")
    bad = nonfinite(r["logits"])
    assert torch.nonzero(bad).flatten().tolist() == [where["graph"]]
    keep = ~bad
    assert torch.equal(r["logits"][keep], clean["logits"][keep])
    assert np.isnan(float(r["logits"][where["graph"]]))


@pytest.mark.parametrize("site", [s for s in SITES if not s[0].startswith("pooling.")], ids=site_id)
def test_node_poison_outside_the_loss_rows(site):
    """Node style with the poisoned node's whole graph outside the loss rows.  The one-node embedding row leaves the loss finite, but
    every weight gradient is still NaN (0 * NaN in the weight GEMMs over the NaN activations) while the head's biases, sums of the
    zero logit gradients, stay finite; a shared parameter makes the loss NaN and every gradient non-finite."""
    g, where = poison_batch("node", 256)
    offs, gi = where["offs"], where["graph"]
    keep = np.zeros(g.num_nodes(), dtype=bool)
    keep[::2] = True
    keep[offs[gi]:offs[gi + 1]] = False
    r = oracle_step(poison(model_state(HIDDEN, "node", 3), site, where), g, "node", torch.from_numpy(np.nonzero(keep)[0]))
    finite = sorted(k for k, v in grad_flags(r["grads"]).items() if not v)
    if site[0] == EMBED:
        assert math.isfinite(float(r["loss"])) and finite == ["output_layer.0.bias", "output_layer.2.bias"]
    else:
        assert math.isnan(float(r["loss"])) and finite == []
