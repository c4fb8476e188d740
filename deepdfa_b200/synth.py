"""Synthetic "Big-Vul-shaped" CFG batches (SURVEY.md §8(d)).

There is no dataset in this environment (the 45 GB preprocessed Big-Vul dump is
absent), so benchmarks and parity tests run on seeded synthetic batches whose
*shape* follows what the reference pipeline hands to the model:

* edges are in DGL orientation after ``dgl.add_self_loop``
  (reference ``dbize_graphs.py:24-25``): one self-loop per node, a reversed
  fall-through chain ``(i+1 -> i)`` (DGL edges are reversed CFG edges,
  ``get_func_graph.sc:53``), and random branch/loop edges until the graph holds
  ``round(edges_per_node * n)`` edges in total (default 2.0 => 150 nodes / 300 edges);
* node features are the four ``_ABS_DATAFLOW_{api,datatype,literal,operator}``
  int64 index vectors (``graphmogrifier.py:76-79``) with 0 = "not a definition"
  (75 % of nodes, shared across subkeys), 1 = UNKNOWN (5 %), else a Zipf-distributed
  known hash in ``[2, input_dim)`` (``dbize_absdf.py:35-42``);
* ``_VULN`` int32 per node (``graphmogrifier.py:81``): all zero except one random
  node in ``vuln_rate`` of the graphs (paper §5.2: 6 %).
"""
from __future__ import annotations

import numpy as np
import torch

from .batched_graph import ABS_DATAFLOW_SUBKEYS, BatchedCFG


def _graph_sizes(rng: np.random.Generator, num_graphs: int, nodes_per_graph: int, variable: bool,
                 sigma: float = 0.6, min_nodes: int = 2, max_nodes: int = 2000) -> np.ndarray:
    if not variable:
        return np.full(num_graphs, nodes_per_graph, dtype=np.int64)
    mu = np.log(nodes_per_graph) - sigma * sigma / 2.0
    n = np.rint(rng.lognormal(mu, sigma, size=num_graphs)).astype(np.int64)
    return np.clip(n, min_nodes, max_nodes)


def make_batch(num_graphs: int = 256, nodes_per_graph: int = 150, edges_per_node: float = 2.0,
               input_dim: int = 1002, seed: int = 0, variable: bool = False,
               vuln_rate: float = 0.06, sizes=None) -> BatchedCFG:
    """Build one batched synthetic CFG batch on the CPU (int64 indices, like DGL)."""
    rng = np.random.default_rng(1234 + seed)
    if sizes is None:
        sizes = _graph_sizes(rng, num_graphs, nodes_per_graph, variable)
    else:
        sizes = np.asarray(sizes, dtype=np.int64)
        num_graphs = len(sizes)
    offs = np.zeros(num_graphs + 1, dtype=np.int64)
    np.cumsum(sizes, out=offs[1:])
    n_total = int(offs[-1])

    srcs, dsts = [], []
    # self loops
    loops = np.arange(n_total, dtype=np.int64)
    # reversed fall-through chain: (i+1 -> i) inside each graph
    is_last = np.zeros(n_total, dtype=bool)
    is_last[offs[1:] - 1] = True
    chain_dst = loops[~is_last]
    chain_src = chain_dst + 1
    # extra branch / loop edges, uniformly inside each graph, to reach the edge budget
    target = np.maximum(np.rint(edges_per_node * sizes).astype(np.int64), 2 * sizes - 1)
    extra = target - (2 * sizes - 1)
    g_of_extra = np.repeat(np.arange(num_graphs), extra)
    n_of_extra = sizes[g_of_extra]
    ex_src = offs[g_of_extra] + (rng.random(g_of_extra.shape[0]) * n_of_extra).astype(np.int64)
    ex_dst = offs[g_of_extra] + (rng.random(g_of_extra.shape[0]) * n_of_extra).astype(np.int64)
    # DGL layout after batch(): edges grouped per graph; inside a graph: CFG edges then self loops
    src = np.concatenate([chain_src, ex_src, loops])
    dst = np.concatenate([chain_dst, ex_dst, loops])
    gid = np.searchsorted(offs[1:], dst, side="right")
    order = np.argsort(gid, kind="stable")
    src, dst = src[order], dst[order]
    bne = np.bincount(gid, minlength=num_graphs)

    # node features
    u = rng.random(n_total)
    is_def = u >= 0.75
    is_unknown = u >= 0.95
    ndata = {}
    combined = np.zeros(n_total, dtype=np.int64)
    for k, key in enumerate(ABS_DATAFLOW_SUBKEYS):
        z = rng.zipf(1.2, size=n_total).astype(np.int64)
        idx = 2 + (z % max(1, input_dim - 2))
        idx = np.where(is_unknown, 1, idx)
        idx = np.where(is_def, idx, 0)
        ndata[f"_ABS_DATAFLOW_{key}"] = torch.from_numpy(idx)
        if k == 0:
            combined = idx
    ndata["_ABS_DATAFLOW"] = torch.from_numpy(combined.copy())

    vuln = np.zeros(n_total, dtype=np.int32)
    is_vuln_graph = rng.random(num_graphs) < vuln_rate
    pick = offs[:-1] + (rng.random(num_graphs) * sizes).astype(np.int64)
    vuln[pick[is_vuln_graph]] = 1
    ndata["_VULN"] = torch.from_numpy(vuln)

    return BatchedCFG(torch.from_numpy(src), torch.from_numpy(dst), torch.from_numpy(sizes.copy()),
                      ndata, torch.from_numpy(bne.astype(np.int64)))


def make_learnable_batch(num_graphs: int, nodes_per_graph: int, seed: int, variable: bool = True, vuln_rate: float = 0.4) -> BatchedCFG:
    """A batch whose graph label can be learned from the node features (``make_batch`` draws labels independently of the
    features, which is right for throughput and parity but leaves nothing to learn): the vulnerable node of a vulnerable graph
    carries api token 7 and operator token 11; 8 % of the clean graphs carry api token 7 on one node as a distractor.  Used by
    the train-both-arms / F1 comparisons (BASELINE configs[2], configs[4])."""
    g = make_batch(num_graphs, nodes_per_graph, seed=seed, variable=variable, vuln_rate=vuln_rate)
    rng = np.random.default_rng(seed)
    vuln = g.ndata["_VULN"].numpy()
    api, op = g.ndata["_ABS_DATAFLOW_api"].numpy(), g.ndata["_ABS_DATAFLOW_operator"].numpy()
    hot = np.nonzero(vuln)[0]
    api[hot] = 7
    op[hot] = 11
    offs = np.concatenate([[0], np.cumsum(g.batch_num_nodes().numpy())])
    labels = np.maximum.reduceat(vuln, offs[:-1])
    for b in np.nonzero(labels == 0)[0]:
        if rng.random() < 0.08:
            api[offs[b] + rng.integers(0, offs[b + 1] - offs[b])] = 7
    return g


def make_edge_cases(input_dim: int = 1002, seed: int = 7) -> BatchedCFG:
    """Tiny ragged batch covering the reference-relevant edge cases (SURVEY.md §4):
    a 1-node graph, a 2-node graph, a 300-node graph, a node with zero in-degree
    (no self loop), a high in-degree hub, and duplicate (multi-)edges."""
    rng = np.random.default_rng(seed)
    sizes = np.array([1, 2, 300, 40, 5], dtype=np.int64)
    g = make_batch(sizes=sizes, input_dim=input_dim, seed=seed)
    src, dst = [t.numpy().copy() for t in g.edges()]
    offs = np.concatenate([[0], np.cumsum(sizes)])
    # graph 3 (40 nodes): hub node offs[3]+0 receives from every node of its graph, twice (duplicates)
    hub = offs[3]
    extra_src = np.concatenate([np.arange(offs[3], offs[4]), np.arange(offs[3], offs[4])])
    extra_dst = np.full_like(extra_src, hub)
    src = np.concatenate([src, extra_src])
    dst = np.concatenate([dst, extra_dst])
    # graph 4 (5 nodes): remove every in-edge of its last node (zero in-degree, no self loop)
    lonely = offs[5] - 1
    keep = dst != lonely
    src, dst = src[keep], dst[keep]
    del rng
    return BatchedCFG(torch.from_numpy(src), torch.from_numpy(dst), g.batch_num_nodes(), g.ndata)


BIGVUL_TAIL = "_all_limitall_1000_limitsubkeys_1000"
_CODE = np.array(["x = 1;", "f(a, b);", 'puts("hi, \\"there\\"");', "if (a)\n{", "return;", "", "nan", "p->q = r[\"k\"];",
                  "/* é ü */", "a\r\nb"])


def write_bigvul_files(root, num_graphs: int, seed: int = 0, mu: float = 3.7, sigma: float = 0.8, big_graph: int = 3000) -> dict:
    """Processed Big-Vul files in the reference's schema under ``root/bigvul`` (dbize.py:104-105: ``nodes.csv`` with an
    unnamed index, ``dgl_id``, ``code``, ``vuln``, ``graph_id``, ``node_id``, ``_label`` and ``edges.csv``; dbize_absdf.py: one shuffled
    ``nodes_feat__ABS_DATAFLOW_<sub>_all_..._fixed.csv`` per subkey): lognormal graph sizes (``mu`` / ``sigma`` of the log, at
    least 2 nodes, graph 0 has ``big_graph`` nodes), about two edge rows per node, unsorted non-contiguous graph ids.  Returns
    the columns as written: {"nodes": {...}, "edges": {...}, "features": {sub: {graph_id, node_id, value}}}."""
    import pandas as pd
    from pathlib import Path
    rng = np.random.default_rng(seed)
    folder = Path(root) / "bigvul"
    folder.mkdir(parents=True, exist_ok=True)
    sizes = np.clip(np.rint(rng.lognormal(mu, sigma, num_graphs)), 2, None).astype(np.int64)
    sizes[0] = big_graph
    gid_of = rng.permutation(np.arange(num_graphs, dtype=np.int64) * 3 + 100)
    N = int(sizes.sum())
    first = np.repeat(np.cumsum(sizes) - sizes, sizes)
    local = np.arange(N) - first
    g_node = np.repeat(gid_of, sizes)
    node_id = 1000 + 4 * local + np.repeat(rng.integers(0, 50, num_graphs), sizes)
    vuln = (rng.random(N) < 0.05).astype(np.int64)
    ecount = 2 * sizes
    Ne = int(ecount.sum())
    eg = np.repeat(np.arange(num_graphs), ecount)
    n_e = sizes[eg]
    src = (rng.random(Ne) * n_e).astype(np.int64)
    dst = (rng.random(Ne) * n_e).astype(np.int64)
    head = np.cumsum(ecount) - ecount
    src[head], dst[head] = sizes - 1, 0                 # every graph names its highest dgl id
    nodes = {"graph_id": g_node, "node_id": node_id, "vuln": vuln}
    edges = {"graph_id": gid_of[eg], "innode": src, "outnode": dst}
    pd.DataFrame({"dgl_id": local, "code": _CODE[rng.integers(0, len(_CODE), N)], "vuln": vuln, "graph_id": g_node,
                  "node_id": node_id, "_label": "CALL"}).to_csv(folder / "nodes.csv")
    pd.DataFrame(edges).to_csv(folder / "edges.csv")
    features = {}
    for sub in ABS_DATAFLOW_SUBKEYS:
        stem = f"_ABS_DATAFLOW_{sub}{BIGVUL_TAIL}"
        order = rng.permutation(N)
        f = {"graph_id": g_node[order], "node_id": node_id[order], "value": rng.integers(0, 1002, N)}
        pd.DataFrame({"graph_id": f["graph_id"], "node_id": f["node_id"], stem: f["value"]}).to_csv(folder / f"nodes_feat_{stem}_fixed.csv")
        features[sub] = f
    return {"nodes": nodes, "edges": edges, "features": features}
