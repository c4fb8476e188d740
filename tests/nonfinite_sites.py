"""Non-finite injection sites shared by tests/test_nonfinite_gpu.py (which runs the kernels) and tests/test_nonfinite_premises.py
(which checks on the CPU what the fp32 oracle does at each site).

A site is one NaN or +-inf written into one place of a model whose other values are finite: one embedding row that exactly one
node of the batch uses, or one element of a parameter.  The reference trains in fp32 and decides there whether a step's
gradients are finite (``detect_anomaly``; GradScaler's skip rule), so the oracle runs in fp32 and the kernels must give the same
non-finite sets: which logits, whether the loss, which parameters' gradients."""
import numpy as np
import torch

from deepdfa_b200 import synth
from oracle import ggnn_oracle as O

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
INPUT_DIM = 1002
STEPS = 3
LAYERS = 2                      # output_layer.0 (hidden, ReLU) and output_layer.2 (last)
POS_WEIGHT = 2.0
NAN, INF = float("nan"), float("inf")

# (engine, hidden_dim): the SIMT engine, the D = 128 tensor-core engine and the wide tensor-core engine at W = 192 (3W = 576 ends
# on a half tile of 64 columns) and W = 256; W = 4 * hidden_dim (concat_all_absdf)
ENGINES = [("simt", 32), ("tcgen05", 32), ("tcgen05", 48), ("tcgen05", 64)]
LAST = f"output_layer.{2 * (LAYERS - 1)}"
GGNN = ["ggnn.linears.0.weight", "ggnn.linears.0.bias", "ggnn.gru.weight_ih", "ggnn.gru.weight_hh", "ggnn.gru.bias_ih",
        "ggnn.gru.bias_hh"]
GATE = ["pooling.gate_nn.weight", "pooling.gate_nn.bias"]
HEAD = ["output_layer.0.weight", "output_layer.0.bias", f"{LAST}.weight", f"{LAST}.bias"]
EMBED = "all_embeddings.api.weight"
# (name, value): the one-node embedding row as NaN, +inf and -inf; one element of every other parameter as NaN
SITES = [(EMBED, NAN), (EMBED, INF), (EMBED, -INF)] + [(k, NAN) for k in GGNN + GATE + HEAD]


def site_id(site):
    name, value = site
    return f"{name}={value}"


def sites(style):
    return [s for s in SITES if style == "graph" or not s[0].startswith("pooling.")]


def case_id(engine, hidden):
    return f"{engine}-W{4 * hidden}"


def poison_batch(style: str, B: int, seed: int = 0):
    """A batch of B graphs (graph style) or B nodes (node style) and the place of its poison: graph `graph`, node `node` in it,
    whose api index is set to `row`, a row of the api table no other node of the batch uses."""
    if style == "graph":
        g = synth.make_batch(B, 12, seed=seed, variable=True, vuln_rate=0.3)
    else:
        sizes = [12] * (B // 12) + ([B % 12] if B % 12 else [])
        g = synth.make_batch(sizes=sizes, seed=seed, vuln_rate=0.3)
        rng = np.random.default_rng(seed)
        g.ndata["_VULN"] = torch.from_numpy((rng.random(B) < 0.2).astype(np.int32))
    offs = np.concatenate([[0], np.cumsum(g.batch_num_nodes().numpy())])
    graph = len(offs) // 3
    node = int(offs[graph] + (offs[graph + 1] - offs[graph]) // 2)
    api = g.ndata["_ABS_DATAFLOW_api"]
    used = set(api.tolist())
    row = max(r for r in range(2, INPUT_DIM) if r not in used)
    api[node] = row
    return g, dict(graph=graph, node=node, row=row, offs=offs)


def element(name: str, shape) -> tuple:
    """The element of a parameter a site poisons (the embedding's is the poison row, set by `poison`)."""
    n = int(np.prod(shape))
    flat = (n // 2 + 1) % n
    return tuple(int(i) for i in np.unravel_index(flat, tuple(shape)))


def poison(state: dict, site, where) -> dict:
    """A copy of a state_dict with the site's value written in."""
    name, value = site
    sd = {k: v.clone() for k, v in state.items()}
    if name == EMBED:
        sd[name][where["row"]] = value
    else:
        sd[name][element(name, sd[name].shape)] = value
    return sd


def model_state(hidden: int, style: str, seed: int) -> dict:
    torch.manual_seed(seed)
    return oracle_model(hidden, style).state_dict()


def oracle_model(hidden: int, style: str):
    return O.OracleFlowGNNGGNN(FEAT, INPUT_DIM, hidden, STEPS, LAYERS, label_style=style, concat_all_absdf=True,
                               positive_weight=POS_WEIGHT)


def oracle_step(state: dict, batch, style: str, rows=None) -> dict:
    """fp32 oracle forward, mean BCE (over `rows` of a node-style batch when given) and backward: logits, loss, {name: grad}."""
    hidden = state["all_embeddings.api.weight"].shape[1]
    o = oracle_model(hidden, style)
    o.load_state_dict(state)
    out = o(batch)
    label = o.get_label(batch)
    if rows is not None:
        rows = torch.as_tensor(rows, dtype=torch.int64)
        loss = o.loss_fn(out[rows], label[rows])
    else:
        loss = o.loss_fn(out, label)
    loss.backward()
    return dict(logits=out.detach(), loss=loss.detach(), grads={k: p.grad.detach().clone() for k, p in o.named_parameters()})


def nonfinite(t: torch.Tensor) -> torch.Tensor:
    return ~torch.isfinite(t)


def grad_flags(grads: dict) -> dict:
    """{name: True if the gradient has a non-finite element}."""
    return {k: bool(nonfinite(g).any()) for k, g in grads.items()}


def touched_rows(where, style: str) -> np.ndarray:
    """Logit rows the poison can reach when it is local to one graph: that graph, or (node style) that graph's nodes."""
    offs = where["offs"]
    g = where["graph"]
    return np.array([g]) if style == "graph" else np.arange(offs[g], offs[g + 1])
