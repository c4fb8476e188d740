"""GPU: the batch producer at Big-Vul size, bit for bit against the exact NumPy collate of tests/arena_batches.py.

One arena of 190 000 synthetic graphs (~10.4 M nodes, ~20.9 M edges, 8 int64 feature vectors, three of them over +-2^62) is
built once.  Checked against the host reference:
  * its own CSR pair (the largest ddfa_build_csr call the library makes), and the same COO as int32 with either CSR skipped;
  * ``arena.batch`` at B = 1 ... 4 097 (1, 2, 3 and 5 passes of arena_scan_kernel's carry) and over all 190 000 graphs, into
    sentinel-filled outputs, for random, descending and one-id-repeated lists; a small arena covers K = 0, no _VULN, a 0-node
    graph and an edgeless graph;
  * ``ddfa_graph_ptr`` from 0 to 190 000 graphs;
  * the C-ABI error contract: a bad id or totals that disagree leave every output untouched and raise the counter;
  * FusedTrainer.step_ids at B = 2 048 and FusedEvaluator.update_ids at B = 4 097 against the same graphs collated on the host,
    bit for bit in deterministic mode."""
import contextlib
import os
import time

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib
from deepdfa_b200 import batched_graph as BG
from deepdfa_b200 import engine as E
from deepdfa_b200._lib import DdfaError, lib, ptr_array
from deepdfa_b200.evaluator import BATCHES, SAMPLES

import arena_batches as A

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
SENT32 = -0x5A5A5A5B                 # 0xA5A5A5A5
SENT64 = -0x5A5A5A5A5A5A5A5B         # 0xA5A5A5A5A5A5A5A5: outside the +-2^62 of the wide keys
SENT_WS = 0xA5


@pytest.fixture(scope="module")
def big():
    g = A.make_arena_graphs(A.ARENA_GRAPHS, 11, A.WIDE_KEYS)
    t0 = time.perf_counter()
    arena = D.GraphArena.from_graphs([g], DEV)           # unbatches the 190 000 graphs, collates them, one ddfa_build_csr
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    # linear in the graph count: an unbatch that scans every edge once per graph would take ~50 min here
    assert seconds < 300, f"GraphArena.from_graphs took {seconds:.0f} s for {A.ARENA_GRAPHS} graphs"
    assert arena.num_graphs == A.ARENA_GRAPHS and len(arena.feats) == 8
    return {"arena": arena, "host": A.host_arena(g), "N": g.num_nodes(), "E": g.num_edges()}


def np_of(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy().astype(np.int64)


# ---- the arena's own CSR ---------------------------------------------------------------------------------------------------
def test_arena_csr_and_the_int32_build_against_lexsort(big):
    arena, host, N, E_ = big["arena"], big["host"], big["N"], big["E"]
    assert N > 10_000_000 and E_ > 20_000_000
    want = A.csr_ref(host["src"], host["dst"], N)
    dg = arena.dg
    got = (dg.indptr, dg.indices[:E_], dg.indptr_t, dg.indices_t[:E_])
    for name, a, b in zip(("indptr", "indices", "indptr_t", "indices_t"), got, want):
        assert np.array_equal(np_of(a), b), name
    assert int(dg._csr_ws.view(torch.int32)[0]) == 0, "no edge dropped"
    assert np.array_equal(np_of(arena.node_off), host["node_off"])
    assert np.array_equal(np_of(arena.vuln), host["ndata"]["_VULN"])
    for k, v in arena.feats.items():
        assert v.dtype == torch.int64 and np.array_equal(v.cpu().numpy(), host["ndata"][k]), k
    # the same COO as int32, once per CSR with the other one skipped
    src = torch.from_numpy(host["src"]).to(torch.int32).to(DEV)
    dst = torch.from_numpy(host["dst"]).to(torch.int32).to(DEV)
    wsb = lib().call("ddfa_build_csr_workspace_bytes", E_, N)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    for side in (0, 1):
        ptr = torch.full((N + 2,), SENT32, dtype=torch.int32, device=DEV)
        idx = torch.full((E_ + 1,), SENT32, dtype=torch.int32, device=DEV)
        fwd, tr = ((ptr, idx), (None, None)) if side == 0 else ((None, None), (ptr, idx))
        lib().call("ddfa_build_csr", src.data_ptr(), dst.data_ptr(), 4, E_, N, E._p(fwd[0]), E._p(fwd[1]), E._p(tr[0]), E._p(tr[1]),
                   ws.data_ptr(), wsb, st)
        torch.cuda.synchronize()
        assert int(ws.view(torch.int32)[0]) == 0
        assert np.array_equal(np_of(ptr[:N + 1]), want[2 * side]) and np.array_equal(np_of(idx[:E_]), want[2 * side + 1])
        assert int(ptr[N + 1]) == SENT32 and int(idx[E_]) == SENT32, "nothing written past the outputs"


# ---- arena.batch against the host collate ------------------------------------------------------------------------------------
def sentinel_outputs(arena, B, N, E_):
    out = arena.alloc_outputs(B, N, E_)
    for k, v in out.items():
        if k == "feats":
            for t in v.values():
                t.fill_(SENT64)
        elif k == "ws":
            v.fill_(SENT_WS)
        elif k != "ids":
            v.fill_(SENT32)
    return out


def assert_batch_equal(ab, out, ref, vuln_key=True):
    N, E_, B = ref["N"], ref["E"], len(ref["batch_num_nodes"])
    ab.check()
    assert (ab.num_nodes(), ab.num_edges(), ab.batch_size) == (N, E_, B)
    assert np.array_equal(np_of(out["graph_ptr"]), ref["graph_ptr"])
    for name in ("indptr", "indptr_t"):
        assert np.array_equal(np_of(out[name]), ref[name]), name
    for name in ("indices", "indices_t"):
        got = np_of(out[name])
        assert np.array_equal(got[:E_], ref[name]), name
        assert (got[E_:] == SENT32).all(), name            # the one-element buffer of an edgeless batch
    assert out["feats"].keys() == {k for k in ref["ndata"] if k != "_VULN"}
    for k, t in out["feats"].items():
        assert np.array_equal(t.cpu().numpy(), ref["ndata"][k]), k
    want_vuln = ref["ndata"]["_VULN"] if vuln_key else np.zeros(N, np.int64)
    assert np.array_equal(np_of(out["vuln"]), want_vuln)
    assert np.array_equal(np_of(ab.batch_num_nodes()), ref["batch_num_nodes"])
    assert np.array_equal(np_of(ab.batch_num_edges()), ref["batch_num_edges"])
    src, dst = ab.edges()
    assert np.array_equal(np_of(src), ref["indices"])
    assert np.array_equal(np_of(dst), np.repeat(np.arange(N), np.diff(ref["indptr"])))


def id_list(kind, B, G, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":                     # with repeats
        return rng.integers(0, G, B)
    if kind == "descending":
        start = int(rng.integers(B - 1, G))
        return np.arange(start, start - B, -1)
    if kind == "one_id":
        return np.full(B, int(rng.integers(0, G)))
    if kind == "all":
        return rng.permutation(G)
    raise ValueError(kind)


CASES = ([("random", B) for B in A.BATCH_SIZES] + [("descending", B) for B in A.BATCH_SIZES] + [("one_id", 3000), ("one_id", 1025)]
         + [("all", A.ARENA_GRAPHS)])


@pytest.mark.parametrize("kind,B", CASES, ids=[f"{k}-{b}" for k, b in CASES])
def test_batch_equals_the_host_collate(big, kind, B):
    arena = big["arena"]
    ids = id_list(kind, B, arena.num_graphs, seed=B)
    ref = A.collate_ref(big["host"], ids)
    out = sentinel_outputs(arena, B, ref["N"], ref["E"])
    ab = arena.batch(ids, out=out)
    torch.cuda.synchronize()
    assert_batch_equal(ab, out, ref)


@pytest.mark.parametrize("keys", [("_VULN",), ("_ABS_DATAFLOW",)], ids=["k0", "no_vuln"])
def test_small_arena_with_empty_graphs(keys):
    singles = A.small_graphs(4, keys)
    arena = D.GraphArena.from_graphs(singles, DEV)
    assert len(arena.feats) == len([k for k in keys if k != "_VULN"])
    host = A.host_arena(BG.batch(singles))
    G = len(singles)
    zero, edgeless = 2, 7
    assert singles[zero].num_nodes() == 0 and singles[edgeless].num_edges() == 0 < singles[edgeless].num_nodes()
    rng = np.random.default_rng(5)
    for ids in ([edgeless], [zero, edgeless, zero], [edgeless, 0, zero, G - 1, 3, 3], rng.integers(0, G, 1025),
                np.arange(G)[::-1]):
        ref = A.collate_ref(host, ids)
        out = sentinel_outputs(arena, len(ids), ref["N"], ref["E"])
        ab = arena.batch(ids, out=out)
        torch.cuda.synchronize()
        assert_batch_equal(ab, out, ref, vuln_key="_VULN" in keys)


# ---- ddfa_graph_ptr ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", A.GRAPH_PTR_SIZES)
def test_graph_ptr_against_cumsum(B):
    rng = np.random.default_rng(B)
    bnn = rng.integers(0, 120, B)
    bnn[rng.random(B) < 0.3] = 0
    if B:
        bnn[-1] = 0
    out = torch.full((B + 2,), SENT32, dtype=torch.int32, device=DEV)
    bnn_d = torch.from_numpy(bnn).to(DEV)
    lib().call("ddfa_graph_ptr", bnn_d.data_ptr() if B else 0, B, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    got = np_of(out)
    assert np.array_equal(got[:B + 1], np.concatenate([[0], np.cumsum(bnn)]))
    assert got[B + 1] == SENT32


# ---- the error contract of ddfa_arena_batch ------------------------------------------------------------------------------------
def produce(arena, ids_dev, B, N, E_, out, ws_bytes=None, num_feats=None):
    """One direct ddfa_arena_batch call (what GraphArena._assemble makes), with the workspace size and feature count overridable."""
    dg = arena.dg
    keys = list(arena.feats)
    fin = [arena.feats[k].data_ptr() for k in keys]
    fout = [out["feats"][k].data_ptr() for k in keys]
    if num_feats is not None and num_feats > len(keys):
        fin, fout = fin + fin[:1] * (num_feats - len(keys)), fout + fout[:1] * (num_feats - len(keys))
    lib().call("ddfa_arena_batch", ids_dev.data_ptr(), B, arena.num_graphs, arena.node_off.data_ptr(), dg.indptr.data_ptr(),
               dg.indices.data_ptr(), dg.indptr_t.data_ptr(), dg.indices_t.data_ptr(), ptr_array(fin),
               len(keys) if num_feats is None else num_feats, arena.vuln.data_ptr(), N, E_, out["graph_ptr"].data_ptr(),
               out["indptr"].data_ptr(), out["indices"].data_ptr(), out["indptr_t"].data_ptr(), out["indices_t"].data_ptr(),
               ptr_array(fout), out["vuln"].data_ptr(), out["ws"].data_ptr(), out["ws"].numel() if ws_bytes is None else ws_bytes,
               torch.cuda.current_stream().cuda_stream)


def assert_untouched(out):
    for k, v in out.items():
        if k == "feats":
            for name, t in v.items():
                assert bool((t == SENT64).all()), name
        elif k not in ("ids", "ws"):
            assert bool((v == SENT32).all()), k


def error_word(out, B):
    torch.cuda.synchronize()
    return int(out["ws"].view(torch.int32)[B + 1])


def test_bad_ids_and_wrong_totals_leave_the_outputs_untouched(big):
    arena = big["arena"]
    G, B = arena.num_graphs, 2049
    rng = np.random.default_rng(8)
    ids = rng.integers(0, G, B)
    bad = ids.copy()
    bad[5], bad[2000] = -1, G                          # both validated by the scan before any arena read
    good = np.delete(ids, [5, 2000])
    ref = A.collate_ref(big["host"], good)
    N, E_ = ref["N"], ref["E"]
    out = sentinel_outputs(arena, B, N, E_)

    # two bad ids, with the totals of the valid ones: the counter's low half counts them, nothing is written
    bad_dev = torch.from_numpy(bad.astype(np.int32)).to(DEV)
    produce(arena, bad_dev, B, N, E_, out)
    err = error_word(out, B)
    assert err & 0xFFFF == 2 and err >> 16 == 0, hex(err)
    assert_untouched(out)
    ab = arena._assemble(bad_dev, B, N, E_, out)       # the same call through the Python layer: check() reports it
    with pytest.raises(DdfaError, match="2 graph id"):
        ab.check()
    assert_untouched(out)

    # valid ids with totals that disagree: bit 16, nothing is written
    good_ids = torch.from_numpy(ids.astype(np.int32)).to(DEV)
    ref_all = A.collate_ref(big["host"], ids)
    for n, e in ((ref_all["N"] + 1, ref_all["E"]), (ref_all["N"], ref_all["E"] - 1)):
        produce(arena, good_ids, B, n, e, out)
        err = error_word(out, B)
        assert err == 1 << 16, hex(err)
        assert_untouched(out)

    # host-side refusals: a workspace 4 bytes short, nine feature vectors
    wsb = lib().call("ddfa_arena_batch_workspace_bytes", B)
    assert out["ws"].numel() == wsb
    with pytest.raises(DdfaError, match="workspace"):
        produce(arena, good_ids, B, ref_all["N"], ref_all["E"], out, ws_bytes=wsb - 4)
    with pytest.raises(DdfaError, match="bad sizes"):
        produce(arena, good_ids, B, ref_all["N"], ref_all["E"], out, num_feats=9)
    torch.cuda.synchronize()
    assert_untouched(out)

    # then a good batch into the same buffers is exact, and graph_ptr past its B - 2 + 1 entries keeps the sentinel
    Bg = B - 2
    gp = out["graph_ptr"]
    out = dict(out, graph_ptr=gp[:Bg + 1])
    ab = arena._assemble(torch.from_numpy(good.astype(np.int32)).to(DEV), Bg, N, E_, out)
    torch.cuda.synchronize()
    assert_batch_equal(ab, out, ref)
    assert bool((gp[Bg + 1:] == SENT32).all())


def test_from_graphs_refuses_nine_feature_vectors():
    singles = A.small_graphs(6)
    for s in singles:
        s.ndata["_EXTRA_0"] = torch.zeros(s.num_nodes(), dtype=torch.int64)
        s.ndata["_EXTRA_1"] = torch.zeros(s.num_nodes(), dtype=torch.int64)
        s.ndata["_EXTRA_2"] = torch.zeros(s.num_nodes(), dtype=torch.int64)
        s.ndata["_EXTRA_3"] = torch.zeros(s.num_nodes(), dtype=torch.int64)
    assert len([k for k in singles[0].ndata if k != "_VULN"]) == 9
    with pytest.raises(ValueError, match="at most 8"):
        D.GraphArena.from_graphs(singles, DEV)


# ---- end to end: trainer and evaluator on arena ids against host batches of the same graphs -----------------------------------
@contextlib.contextmanager
def det_mode():
    prev = os.environ.get("DDFA_DETERMINISTIC")
    os.environ["DDFA_DETERMINISTIC"] = "1"
    try:
        yield
    finally:
        if prev is None:
            os.environ.pop("DDFA_DETERMINISTIC")
        else:
            os.environ["DDFA_DETERMINISTIC"] = prev
        _lib.apply_deterministic_mode()


def new_module(seed=7):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine="tcgen05").to(DEV)


def test_trainer_step_ids_equals_host_steps(big):
    arena = big["arena"]
    rng = np.random.default_rng(21)
    ids = [rng.integers(0, arena.num_graphs, 2048) for _ in range(3)]
    host = [A.ref_batch(A.collate_ref(big["host"], i)) for i in ids]
    runs = []
    with det_mode():
        for mode in ("ids", "host"):
            tr = D.FusedTrainer(new_module(), use_cuda_graph=True)
            losses = [float(tr.step_ids(arena, i) if mode == "ids" else tr.step(h)) for i, h in zip(ids, host)]
            torch.cuda.synchronize()
            runs.append((losses, [t.detach().clone() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]))
    (la, sa), (lb, sb) = runs
    assert la == lb, (la, lb)
    assert all(torch.equal(x, y) for x, y in zip(sa, sb))


def test_evaluator_update_ids_equals_host_updates(big):
    arena = big["arena"]
    rng = np.random.default_rng(22)
    ids = [rng.integers(0, arena.num_graphs, 4097) for _ in range(5)]
    host = [A.ref_batch(A.collate_ref(big["host"], i)) for i in ids]
    m = new_module(3)
    states = []
    with det_mode():
        for mode in ("ids", "host"):
            ev = D.FusedEvaluator(m)
            for i, h in zip(ids, host):
                ev.update_ids(arena, i) if mode == "ids" else ev.update(h)
            torch.cuda.synchronize()
            states.append(ev.state().clone())
    assert torch.equal(states[0], states[1]), (states[0], states[1])
    assert states[0][SAMPLES].item() == 5 * 4097 and states[0][BATCHES].item() == 5
