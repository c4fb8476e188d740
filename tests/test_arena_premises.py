"""Without a GPU: the exact host collate of tests/arena_batches.py against batched_graph.batch, the launch shapes
tests/test_arena_scale_gpu.py is written for, and batched_graph.unbatch against its former per-graph formulation."""
import numpy as np
import pytest
import torch

from deepdfa_b200 import batched_graph as BG
from deepdfa_b200 import synth

import arena_batches as A


def lexsorted_csr(g: BG.BatchedCFG):
    src, dst = (t.numpy().astype(np.int64) for t in g.edges())
    return A.csr_ref(src, dst, g.num_nodes())


def test_csr_ref_against_per_node_lists():
    rng = np.random.default_rng(0)
    N = 37
    src, dst = rng.integers(0, N, 300), rng.integers(0, N, 300)
    src[:20], dst[:20] = 5, 9                  # duplicate edges
    indptr, indices, indptr_t, indices_t = A.csr_ref(src, dst, N)
    for v in range(N):
        assert indices[indptr[v]:indptr[v + 1]].tolist() == sorted(src[dst == v].tolist())
        assert indices_t[indptr_t[v]:indptr_t[v + 1]].tolist() == sorted(dst[src == v].tolist())
    assert indptr[0] == 0 and indptr[-1] == 300 and indptr_t[-1] == 300


@pytest.mark.parametrize("keys", [None, ("_VULN",), ("_ABS_DATAFLOW",)], ids=["all", "vuln_only", "no_vuln"])
def test_collate_ref_equals_batch_plus_lexsort(keys):
    singles = A.small_graphs(3, keys)
    G = len(singles)
    assert [s.num_nodes() for s in singles].count(0) == 2 and sum(s.num_nodes() > 0 and s.num_edges() == 0 for s in singles) == 1
    host = A.host_arena(BG.batch(singles))
    rng = np.random.default_rng(1)
    for ids in ([2], [7], [0, 0, 0], list(range(G))[::-1], rng.integers(0, G, 200).tolist(), [G - 1, 2, 7, 2, G - 1, 4]):
        ref = A.collate_ref(host, ids)
        want = BG.batch([singles[i] for i in ids])
        assert np.array_equal(ref["batch_num_nodes"], want.batch_num_nodes().numpy())
        assert np.array_equal(ref["batch_num_edges"], want.batch_num_edges().numpy())
        assert np.array_equal(ref["graph_ptr"], np.concatenate([[0], np.cumsum(want.batch_num_nodes().numpy())]))
        assert (ref["N"], ref["E"]) == (want.num_nodes(), want.num_edges())
        assert np.array_equal(ref["src"], want.edges()[0].numpy()) and np.array_equal(ref["dst"], want.edges()[1].numpy())
        for a, b in zip((ref["indptr"], ref["indices"], ref["indptr_t"], ref["indices_t"]), lexsorted_csr(want)):
            assert a.dtype == np.int64 and np.array_equal(a, b)
        assert set(ref["ndata"]) == set(want.ndata)
        for k, v in want.ndata.items():
            assert ref["ndata"][k].dtype == v.numpy().dtype and np.array_equal(ref["ndata"][k], v.numpy()), k
        back = A.ref_batch(ref)
        assert all(torch.equal(a, b) for a, b in zip(back.edges(), want.edges()))


def test_wide_keys_need_64_bits():
    g = A.make_arena_graphs(50, 0, A.WIDE_KEYS)
    assert len([k for k in g.ndata if k != "_VULN"]) == 8
    for k in A.WIDE_KEYS:
        v = g.ndata[k]
        assert v.dtype == torch.int64
        assert bool((v.abs() >= 2 ** 32).float().mean() > 0.99)
        assert bool((v < 0).any()) and bool((v > 0).any())


def test_batch_sizes_reach_the_scan_passes():
    """arena_scan_kernel and graph_ptr_kernel run one 1 024-thread CTA that carries its prefix from pass to pass."""
    passes = {B: A.scan_passes(B) for B in A.BATCH_SIZES}
    assert set(passes.values()) == {1, 2, 3, 5}
    assert passes[1024] == 1 and passes[1025] == 2 and passes[2048] == 2 and passes[2049] == 3
    assert A.scan_passes(A.ARENA_GRAPHS) > 180
    assert {A.scan_passes(B) for B in A.GRAPH_PTR_SIZES} >= {0, 1, 2, 5} and max(A.GRAPH_PTR_SIZES) == A.ARENA_GRAPHS
    # FusedEvaluator.update_ids at B = 4 097: the graph metric kernel's warps stride over the batch
    assert max(A.BATCH_SIZES) > A.METRIC_GRAPHS


# ---- unbatch ---------------------------------------------------------------------------------------------------------------
def unbatch_per_graph(g):
    """batched_graph.unbatch as it was before it sorted once: one scan over all edges per graph."""
    bnn = g.batch_num_nodes().tolist()
    out = []
    n0 = 0
    src, dst = g.edges()
    ptr = torch.tensor([0] + bnn).cumsum(0)
    gid = torch.bucketize(dst.cpu().to(torch.int64), ptr[1:], right=True)
    for b, nn_ in enumerate(bnn):
        sel = (gid == b).nonzero().squeeze(-1).to(src.device)
        nd = {k: v[n0:n0 + nn_] for k, v in g.ndata.items()}
        out.append(BG.BatchedCFG(src[sel] - n0, dst[sel] - n0, torch.tensor([nn_]), nd, torch.tensor([int(sel.numel())])))
        n0 += nn_
    return out


def shuffled_batch(dtype):
    singles = A.small_graphs(5) + BG.unbatch(synth.make_batch(40, 30, seed=6, variable=True))
    g = BG.batch(singles)
    src, dst = g.edges()
    perm = torch.from_numpy(np.random.default_rng(2).permutation(src.numel()))
    src, dst = src[perm], dst[perm]
    # one edge whose dst lies past the last node: it belongs to no graph and both forms drop it
    src, dst = torch.cat([src, torch.tensor([0])]), torch.cat([dst, torch.tensor([g.num_nodes() + 3])])
    return BG.BatchedCFG(src.to(dtype), dst.to(dtype), g.batch_num_nodes(), g.ndata), singles


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32])
def test_unbatch_equals_the_per_graph_form(dtype):
    g, singles = shuffled_batch(dtype)
    assert 0 in g.batch_num_nodes().tolist()
    got, want = BG.unbatch(g), unbatch_per_graph(g)
    assert len(got) == len(want) == g.batch_size
    for a, b, s in zip(got, want, singles):
        assert a.num_nodes() == b.num_nodes() == s.num_nodes()
        assert torch.equal(a.batch_num_nodes(), b.batch_num_nodes()) and torch.equal(a.batch_num_edges(), b.batch_num_edges())
        for x, y in zip(a.edges(), b.edges()):
            assert x.dtype == y.dtype == dtype and torch.equal(x, y)
        assert a.ndata.keys() == b.ndata.keys() and all(torch.equal(a.ndata[k], b.ndata[k]) for k in a.ndata)
        # the same edges as the graph batched in, in the shuffled order
        key = lambda e: sorted(zip(e[0].tolist(), e[1].tolist()))
        assert key(a.edges()) == key(s.edges())
