"""Arenas and an exact host collate for the batch producer, shared by tests/test_arena_scale_gpu.py (which holds
``ddfa_arena_batch``, ``ddfa_build_csr`` and ``ddfa_graph_ptr`` to it at dataset size) and tests/test_arena_premises.py (which
checks it, and the launch shapes the GPU tests are written for, without a GPU).

``collate_ref`` is NumPy only: it never calls ``ddfa_build_csr`` or ``batched_graph.batch``, so a fault shared by the library's
collate and its CSR build cannot hide in the reference."""
import numpy as np
import torch

from deepdfa_b200.batched_graph import BatchedCFG, unbatch
from deepdfa_b200 import synth

# Launch shapes of csrc/arena.cu, csrc/csr_build.cu and csrc/eval_metrics.cu
SCAN_THREADS = 1024          # arena_scan_kernel / graph_ptr_kernel: one CTA, 1 024 graphs per pass, a carry between passes
METRIC_GRAPHS = 264 * 8      # graph_metrics_kernel: 264 CTAs x 8 warps, one warp per graph; past this the grid strides

ARENA_GRAPHS = 190_000       # about the Big-Vul function count: ~10^7 nodes, ~2 x 10^7 edges
BATCH_SIZES = (1, 1023, 1024, 1025, 2048, 2049, 4097)
GRAPH_PTR_SIZES = (0, 1, 1023, 1024, 1025, 4097, ARENA_GRAPHS)
WIDE_KEYS = ("_WIDE_0", "_WIDE_1", "_WIDE_2")    # three int64 keys past the synthetic five: K = 8, the producer's maximum


def scan_passes(B: int) -> int:
    return -(-B // SCAN_THREADS)


def make_arena_graphs(G: int, seed: int, wide_keys=()) -> BatchedCFG:
    """``G`` synthetic graphs of ~55 nodes as one batch; every key of ``wide_keys`` adds an int64 node vector drawn over
    +-2^62, so a copy that keeps 32 bits of it is caught."""
    g = synth.make_batch(G, 55, variable=True, vuln_rate=0.3, seed=seed)
    rng = np.random.default_rng(seed + 77)
    for k in wide_keys:
        g.ndata[k] = torch.from_numpy(rng.integers(-2 ** 62, 2 ** 62, g.num_nodes(), dtype=np.int64))
    return g


def small_graphs(seed: int, keys=None) -> list:
    """Single graphs of 1 to 150 nodes with a 0-node graph and an edgeless 9-node graph among them; ``keys`` keeps only those
    ndata keys (``()`` keeps none)."""
    g = synth.make_batch(sizes=[5, 1, 150, 12, 2, 64, 9, 33], seed=seed, vuln_rate=0.5)
    singles = unbatch(g)
    if keys is not None:
        singles = [BatchedCFG(*s.edges(), s.batch_num_nodes(), {k: s.ndata[k] for k in keys}, s.batch_num_edges()) for s in singles]
    empty = torch.empty(0, dtype=torch.int64)
    zero = BatchedCFG(empty, empty, torch.tensor([0]), {k: v[:0] for k, v in singles[0].ndata.items()}, torch.tensor([0]))
    s = singles[6]
    edgeless = BatchedCFG(empty, empty, s.batch_num_nodes(), s.ndata, torch.tensor([0]))
    return singles[:2] + [zero] + singles[2:6] + [edgeless] + singles[7:] + [zero]


def host_arena(g: BatchedCFG) -> dict:
    """The arena's contents as int64 NumPy arrays: ``node_off`` [G+1], the edges grouped by the graph owning their dst (each
    graph's edges in their stored order, node ids global) with ``edge_off`` [G+1], and ``ndata``."""
    bnn = g.batch_num_nodes().numpy().astype(np.int64)
    node_off = np.concatenate([[0], np.cumsum(bnn)]).astype(np.int64)
    src, dst = (t.numpy().astype(np.int64) for t in g.edges())
    gid = np.searchsorted(node_off[1:], dst, side="right")
    order = np.argsort(gid, kind="stable")
    edge_off = np.concatenate([[0], np.cumsum(np.bincount(gid, minlength=len(bnn))[: len(bnn)])]).astype(np.int64)
    return {"node_off": node_off, "edge_off": edge_off, "src": src[order], "dst": dst[order],
            "ndata": {k: v.numpy() for k, v in g.ndata.items()}}


def _ranges(starts: np.ndarray, lengths: np.ndarray) -> np.ndarray:
    """concat(arange(s, s + n) for s, n in zip(starts, lengths)), int64."""
    total = int(lengths.sum())
    first = np.repeat(np.cumsum(lengths) - lengths, lengths)
    return np.repeat(starts, lengths) + (np.arange(total, dtype=np.int64) - first)


def csr_ref(src: np.ndarray, dst: np.ndarray, N: int):
    """CSR by destination and CSR by source, neighbour lists sorted by id: (indptr, indices, indptr_t, indices_t), int64."""
    o = np.lexsort((src, dst))
    ot = np.lexsort((dst, src))
    indptr = np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=N))]).astype(np.int64)
    indptr_t = np.concatenate([[0], np.cumsum(np.bincount(src, minlength=N))]).astype(np.int64)
    return indptr, src[o], indptr_t, dst[ot]


def collate_ref(arena_host: dict, ids) -> dict:
    """The batch of graphs ``ids`` (repeats allowed) in that order, as ``dgl.batch`` + a CSR build give it, all int64."""
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    node_off, edge_off = arena_host["node_off"], arena_host["edge_off"]
    nn_ = node_off[ids + 1] - node_off[ids]
    ne_ = edge_off[ids + 1] - edge_off[ids]
    graph_ptr = np.concatenate([[0], np.cumsum(nn_)]).astype(np.int64)
    N = int(graph_ptr[-1])
    nodes = _ranges(node_off[ids], nn_)
    edges = _ranges(edge_off[ids], ne_)
    shift = np.repeat(graph_ptr[:-1] - node_off[ids], ne_)        # per copy: its first batch node minus its first arena node
    src = arena_host["src"][edges] + shift
    dst = arena_host["dst"][edges] + shift
    indptr, indices, indptr_t, indices_t = csr_ref(src, dst, N)
    ndata = {k: v[nodes] for k, v in arena_host["ndata"].items()}
    return {"graph_ptr": graph_ptr, "batch_num_nodes": nn_, "batch_num_edges": ne_, "N": N, "E": int(ne_.sum()),
            "src": src, "dst": dst, "indptr": indptr, "indices": indices, "indptr_t": indptr_t, "indices_t": indices_t,
            "ndata": ndata}


def ref_batch(ref: dict) -> BatchedCFG:
    """``collate_ref``'s result as a host BatchedCFG (COO in collate order), for the trainer and evaluator paths."""
    nd = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in ref["ndata"].items()}
    return BatchedCFG(torch.from_numpy(ref["src"]), torch.from_numpy(ref["dst"]), torch.from_numpy(ref["batch_num_nodes"]), nd,
                      torch.from_numpy(ref["batch_num_edges"]))
