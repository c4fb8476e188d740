"""GPU: the encoder cache.

  1. Its contents, bit for bit against ``engine.forward(training=False, head=False)`` of differently composed batches (shuffled ids,
     each graph alone) — the premise that a node's h_T does not depend on the other graphs of its batch — for the SIMT engine at
     W = 32 and the tensor-core engine at W = 128 and 256, built with 1, 7 and 1 024 graphs per pass, over an arena with 0-node
     and edgeless graphs.
  2. ``ddfa_cache_batch`` against an exact torch index gather, into sentinel-filled outputs: B = 1 ... 4 097 with repeated and
     reversed ids; the error contract (a bad id, N +- 1, a short workspace leave every output untouched); and one Big-Vul-size
     case (190 000 graphs, ~10.4 M nodes, D = 128: each plane past 2^32 bytes).
  3. FusedTrainer.step_ids(cache, ids) against step_ids(arena, ids) on the same frozen module, bit for bit in deterministic mode:
     losses, parameters, Adam moments and grad_norm, graph and node style, with accumulation and clipping, captured and eager.
  4. FusedEvaluator.update_ids and 5. FusedPredictor.predict_ids over the cache against the arena, exactly.
  6. After the encoder changes, the next call over the cache raises instead of replaying a captured graph.
  7. An owner reused across a rebuilt cache lets the old cache go (its planes are freed) and captures the new one.
  8. Two NCCL ranks, graph and node style: step_ids(cache) equals step_ids(arena) on every rank (skipped below two GPUs)."""
import contextlib
import json
import os

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200 import engine as E
from deepdfa_b200.module import _ENGINES

import arena_batches as A

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
SENT32 = -0x5A5A5A5B                 # 0xA5A5A5A5
SENT_WS = 0xA5


@contextlib.contextmanager
def det_mode(on=True):
    prev = os.environ.get("DDFA_DETERMINISTIC")
    os.environ["DDFA_DETERMINISTIC"] = "1" if on else "0"
    try:
        yield
    finally:
        if prev is None:
            os.environ.pop("DDFA_DETERMINISTIC")
        else:
            os.environ["DDFA_DETERMINISTIC"] = prev
        _lib.apply_deterministic_mode()


@pytest.fixture(scope="module")
def arena():
    """~90 graphs: 80 synthetic ones of ~40 nodes and the small set of tests/arena_batches.py (a 0-node graph at three places,
    an edgeless graph, 1 to 150 nodes)."""
    big = synth.make_batch(80, 40, seed=31, variable=True, vuln_rate=0.3)
    small = A.small_graphs(5)
    return D.GraphArena.from_graphs(small[:5] + [big] + small[5:], DEV)


def module(engine="tcgen05", hidden=32, style="graph", seed=3, steps=4, freeze=True, **kw):
    torch.manual_seed(seed)
    m = D.FlowGNNGGNNModule(FEAT, 1002, hidden, steps, 2, label_style=style, concat_all_absdf=True, positive_weight=2.0, engine=engine,
                            **kw).to(DEV)
    if freeze:
        for name, p in m.named_parameters():
            if not name.startswith(("output_layer.", "pooling.")):
                p.requires_grad_(False)
    return m


def node_range(arena, ids):
    off = np.concatenate([[0], np.cumsum(arena.nodes_per_graph)])
    return np.concatenate([np.arange(off[i], off[i + 1]) for i in ids]).astype(np.int64)


def forward_rows(m, arena, ids):
    """x and h_T of the batch ``ids`` from the module's GGNN forward in its inference form."""
    b = arena.batch(ids)
    params = E.ParamPack.from_flat_list([p.data for p in m.param_list()], len(m._tables()), m._num_layers)
    idx = E.node_indices(b, m.concat_all_absdf, m.feature_keys["feature"], DEV)
    x, h, _ = E.forward(params, E.prepare_graph(b, DEV), idx, m.hparams.n_steps, training=False, engine=_ENGINES[m.engine], head=False)
    return x.clone(), h.clone()


# ---- 1. the cache's contents --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine,hidden", [("simt", 8), ("tcgen05", 32), ("tcgen05", 64)], ids=["simt-W32", "tc-W128", "tc-W256"])
def test_cache_rows_do_not_depend_on_the_batch(arena, engine, hidden):
    m = module(engine, hidden)
    G = arena.num_graphs
    caches = [D.EncoderCache(m, arena, graphs_per_batch=gpb) for gpb in (1, 7, 1024)]
    c = caches[0]
    assert c.h.shape == (c.num_nodes, 4 * hidden) and c.nbytes == 2 * c.num_nodes * 4 * hidden * 4
    for other in caches[1:]:
        assert torch.equal(other.h, c.h) and torch.equal(other.x, c.x)
    assert torch.isfinite(c.h).all()
    perm = np.random.default_rng(0).permutation(G)
    x, h = forward_rows(m, arena, perm)
    rows = torch.from_numpy(node_range(arena, perm)).to(DEV)
    assert torch.equal(x, c.x[rows]) and torch.equal(h, c.h[rows]), \
        f"shuffled batch: max |dh| {float((h - c.h[rows]).abs().max()):.3e}"
    off = np.concatenate([[0], np.cumsum(arena.nodes_per_graph)])
    for i in range(G):
        if off[i + 1] == off[i]:
            continue
        x, h = forward_rows(m, arena, [i])
        assert torch.equal(x, c.x[off[i]:off[i + 1]]) and torch.equal(h, c.h[off[i]:off[i + 1]]), f"graph {i} alone"


# ---- 2. ddfa_cache_batch -----------------------------------------------------------------------------------------------------
def planes(sizes, D_, seed=0):
    """node_off, vuln and the two planes of a synthetic cache whose every 32-bit word is distinct (bit patterns, NaNs included)."""
    n_all = int(np.sum(sizes))
    node_off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(DEV)
    row = torch.arange(n_all, dtype=torch.int32, device=DEV)[:, None]
    col = torch.arange(D_, dtype=torch.int32, device=DEV)[None, :]
    h = (row * 131 + col + seed).view(torch.float32) if D_ <= 131 else (row * D_ + col).view(torch.float32)
    x = (-(row * 131 + col) - 1 - seed).view(torch.float32) if D_ <= 131 else (-(row * D_ + col) - 1).view(torch.float32)
    vuln = (torch.arange(n_all, dtype=torch.int32, device=DEV) * 7 + seed) % 5
    return node_off, vuln, h.contiguous(), x.contiguous()


def run_cache_batch(node_off, vuln, h, x, ids, N, pad=3, ws_bytes=None):
    """ddfa_cache_batch into sentinel-filled outputs ``pad`` rows / words longer than needed; returns (rc, outputs, ws)."""
    L = _lib.lib()
    B, D_ = len(ids), h.shape[1]
    ids_t = torch.tensor(np.asarray(ids, dtype=np.int32), device=DEV)
    out = {"graph_ptr": torch.full((B + 1 + pad,), SENT32, dtype=torch.int32, device=DEV),
           "vuln": torch.full((max(N, 0) + pad,), SENT32, dtype=torch.int32, device=DEV),
           "h": torch.full((max(N, 0) + pad, D_), SENT32, dtype=torch.int32, device=DEV).view(torch.float32),
           "x": torch.full((max(N, 0) + pad, D_), SENT32, dtype=torch.int32, device=DEV).view(torch.float32)}
    need = L.call("ddfa_cache_batch_workspace_bytes", B)
    ws = torch.full((need,), SENT_WS, dtype=torch.uint8, device=DEV)
    rc = L.raw("ddfa_cache_batch")(ids_t.data_ptr(), B, node_off.numel() - 1, node_off.data_ptr(), vuln.data_ptr(), h.data_ptr(),
                                   x.data_ptr(), h.shape[0], D_, N, out["graph_ptr"].data_ptr(), out["vuln"].data_ptr(),
                                   out["h"].data_ptr(), out["x"].data_ptr(), ws.data_ptr(), need if ws_bytes is None else ws_bytes,
                                   torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, out, ws


def expected(node_off, vuln, h, x, ids):
    off = node_off.cpu().numpy().astype(np.int64)
    sizes = off[1:] - off[:-1]
    rows = torch.from_numpy(np.concatenate([np.arange(off[i], off[i + 1]) for i in ids] + [np.zeros(0, np.int64)])).to(DEV)
    gp = np.concatenate([[0], np.cumsum(sizes[np.asarray(ids)])]).astype(np.int32)
    return torch.from_numpy(gp).to(DEV), vuln[rows], h.view(torch.int32)[rows], x.view(torch.int32)[rows]


def assert_gathered(out, want, B, N, pad=3):
    gp, v, h, x = want
    assert torch.equal(out["graph_ptr"][:B + 1], gp)
    assert torch.equal(out["vuln"][:N], v)
    assert torch.equal(out["h"].view(torch.int32)[:N], h) and torch.equal(out["x"].view(torch.int32)[:N], x)
    for k in ("graph_ptr", "vuln", "h", "x"):                         # nothing past the batch is written
        tail = out[k].view(torch.int32)[-pad:]
        assert bool((tail == SENT32).all()), k


def assert_untouched(out):
    for k, t in out.items():
        assert bool((t.view(torch.int32) == SENT32).all()), k


@pytest.fixture(scope="module")
def small_planes():
    rng = np.random.default_rng(4)
    sizes = rng.integers(0, 90, 5000)
    sizes[::37] = 0
    sizes[11] = 3000                                                   # one graph of 3 000 nodes: many slices
    return {D_: planes(sizes, D_) for D_ in (32, 128, 512)}


@pytest.mark.parametrize("D_", [32, 128, 512])
@pytest.mark.parametrize("B", [1, 1023, 1024, 1025, 4097])
def test_gather_against_torch_index(small_planes, D_, B):
    node_off, vuln, h, x = small_planes[D_]
    G = node_off.numel() - 1
    sizes = (node_off[1:] - node_off[:-1]).cpu().numpy()
    rng = np.random.default_rng(B)
    for ids in (rng.integers(0, G, B),                                  # random, repeats
                np.arange(G - 1, G - 1 - B, -1) % G,                     # reversed
                np.full(B, 11 if B * 3000 * D_ <= 2 ** 31 else 12)):    # one id repeated (the 3 000-node one while it fits)
        N = int(sizes[ids].sum())
        rc, out, ws = run_cache_batch(node_off, vuln, h, x, ids, N)
        assert rc == 0
        assert int(ws[:4].view(torch.int32)) == 0
        assert_gathered(out, expected(node_off, vuln, h, x, ids), B, N)


def test_error_contract_leaves_outputs_untouched(small_planes):
    node_off, vuln, h, x = small_planes[128]
    G = node_off.numel() - 1
    sizes = (node_off[1:] - node_off[:-1]).cpu().numpy()
    ids = np.arange(0, 2000, 3)
    N = int(sizes[ids].sum())
    for bad, count in ((G, 1), (-1, 1), (2 ** 31 - 1, 1)):
        b = ids.copy()
        b[5] = bad
        b[-1] = bad
        rc, out, ws = run_cache_batch(node_off, vuln, h, x, b, N)
        assert rc == 0 and int(ws[:4].view(torch.int32)) & 0xFFFF == 2 * count
        assert_untouched(out)
    for n in (N - 1, N + 1):
        rc, out, ws = run_cache_batch(node_off, vuln, h, x, ids, n)
        assert rc == 0 and int(ws[:4].view(torch.int32)) == 1 << 16
        assert_untouched(out)
    need = _lib.lib().call("ddfa_cache_batch_workspace_bytes", len(ids))
    rc, out, ws = run_cache_batch(node_off, vuln, h, x, ids, N, ws_bytes=need - 1)
    assert rc == -4 and bool((ws == SENT_WS).all())
    assert_untouched(out)
    rc, out, _ = run_cache_batch(node_off, vuln, h, x, ids, N)         # and the same call with good arguments goes through
    assert rc == 0
    assert_gathered(out, expected(node_off, vuln, h, x, ids), len(ids), N)


def test_big_vul_size_offsets_past_2_32_bytes():
    """190 000 graphs (~10.4 M nodes), D = 128: each plane 5.3 GB, so the last graphs' rows start past 2^32 bytes."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    rng = np.random.default_rng(190)
    sizes = rng.integers(1, 109, A.ARENA_GRAPHS)                         # mean ~55 nodes: Big-Vul's ~10^7 nodes
    node_off, vuln, h, x = planes(sizes, 128)
    n_all = int(sizes.sum())
    assert n_all > 10_000_000 and 2 * n_all * 128 * 4 > 10.5e9 and (n_all - 200) * 128 * 4 > 2 ** 32
    G = A.ARENA_GRAPHS
    for ids in (np.arange(G - 1, G - 4098, -1),                          # the last 4 097 graphs, reversed
                rng.integers(0, G, 4097),
                np.array([G - 1, 0, G - 1])):
        N = int(sizes[ids].sum())
        rc, out, ws = run_cache_batch(node_off, vuln, h, x, ids, N)
        assert rc == 0 and int(ws[:4].view(torch.int32)) == 0
        assert_gathered(out, expected(node_off, vuln, h, x, ids), len(ids), N)
    peak = torch.cuda.max_memory_allocated() - base
    print(json.dumps({"big_vul_cache_batch": {"graphs": G, "nodes": n_all, "D": 128, "cache_gib": round(2 * n_all * 512 / 2 ** 30, 2),
                                              "peak_gib": round(peak / 2 ** 30, 2)}}))
    del node_off, vuln, h, x
    torch.cuda.empty_cache()


# ---- 3. the trainer --------------------------------------------------------------------------------------------------------
def id_lists(arena, n, seed):
    """``n`` id lists of 5 to 24 graphs; list i + 3 repeats list i, so captured slots are replayed."""
    rng = np.random.default_rng(seed)
    base = [rng.choice(arena.num_graphs, int(rng.integers(5, 25)), replace=bool(i % 2)) for i in range(3)]
    return [base[i % 3] for i in range(n)]


TRAIN_CASES = {
    "graph": dict(style="graph"),
    "graph-acc3": dict(style="graph", tr=dict(accumulate_grad_batches=3)),
    "graph-clip": dict(style="graph", tr=dict(max_grad_norm=0.05, skip_nonfinite=True, track_metrics=True)),
    "graph-adamw-simt": dict(style="graph", engine="simt", hidden=8, tr=dict(decoupled_weight_decay=True)),
    "node": dict(style="node", factor=1.0),
    "node-acc3-clip": dict(style="node", factor=2.0, tr=dict(accumulate_grad_batches=3, max_grad_norm=0.05, track_metrics=True)),
}


@pytest.mark.parametrize("captured", [True, False], ids=["captured", "eager"])
@pytest.mark.parametrize("case", list(TRAIN_CASES))
def test_trainer_steps_match_the_arena_step(arena, case, captured):
    cfg = TRAIN_CASES[case]
    style, tr_kw = cfg["style"], cfg.get("tr", {})
    kw = dict(undersample_node_on_loss_factor=cfg["factor"]) if "factor" in cfg else {}
    with det_mode(True):
        runs = []
        for source in ("arena", "cache"):
            m = module(cfg.get("engine", "tcgen05"), cfg.get("hidden", 32), style, **kw)
            tr = D.FusedTrainer(m, use_cuda_graph=captured, node_sample_seed=5, **tr_kw)
            src = arena if source == "arena" else D.EncoderCache(m, arena)   # after the trainer: its flat buffer holds the params
            losses, norms = [], []
            for ids in id_lists(arena, 8, 17):
                losses.append(tr.step_ids(src, ids).clone())
                if tr.grad_norm is not None:
                    norms.append(tr.grad_norm.clone())
            tr.flush()
            torch.cuda.synchronize()
            runs.append(dict(loss=torch.cat(losses), norm=torch.cat(norms) if norms else None, p=tr.flat_p.clone(),
                             m=tr.exp_avg.clone(), v=tr.exp_avg_sq.clone(), step=int(tr.step_count), metrics=tr.metrics() if tr.track_metrics else None,
                             rows=tr.last_loss_rows() if style == "node" else None))
        a, c = runs
        assert torch.equal(a["loss"], c["loss"]), (a["loss"], c["loss"])
        assert torch.equal(a["p"], c["p"]) and torch.equal(a["m"], c["m"]) and torch.equal(a["v"], c["v"])
        assert a["step"] == c["step"] > 0
        if a["norm"] is not None:
            assert torch.equal(a["norm"], c["norm"])
        assert a["metrics"] == c["metrics"]
        if style == "node":
            assert torch.equal(a["rows"], c["rows"])


def test_cached_step_slots_count_against_max_graph_shapes(arena):
    m = module()
    tr = D.FusedTrainer(m, use_cuda_graph=True, max_graph_shapes=1)
    cache = D.EncoderCache(m, arena)
    tr.step_ids(cache, [1, 2, 3])
    tr.step_ids(cache, [4, 5])                       # a second shape: no slot left, eager over fresh outputs
    assert len(tr._stream_slots) == 1 and next(iter(tr._stream_slots))[:2] == ("cache", id(cache))
    tr.step_ids(arena, [1, 2, 3])                    # and the arena's shape too
    assert len(tr._stream_slots) == 1


# ---- 4. the evaluator --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("style,statements", [("graph", None), ("graph", "attention"), ("node", "probability")])
def test_evaluator_over_the_cache_matches_the_arena(arena, style, statements):
    m = module(style=style, freeze=False)
    cache = D.EncoderCache(m, arena)
    out = []
    for src in (arena, cache):
        ev = D.FusedEvaluator(m, max_predictions=40000, statements=statements)
        scores = []
        for ids in id_lists(arena, 7, 23):
            ev.update_ids(src, ids)
            if statements:
                scores.append(ev.last_scores().clone())
        probs, labels = ev.predictions()
        out.append((ev.compute(), probs.clone(), labels.clone(), torch.cat(scores) if scores else None))
    (ca, pa, la, sa), (cc, pc, lc, sc) = out
    assert ca == cc
    assert torch.equal(pa, pc) and torch.equal(la, lc)
    if statements:
        assert torch.equal(sa, sc)


# ---- 5. the predictor --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("style,statements,kw", [("graph", "attention", {}), ("node", "probability", {}),
                                                 ("graph", "attention", {"encoder_mode": True}), ("graph", None, {"encoder_mode": True})],
                         ids=["graph-attention", "node-probability", "encoder-attention", "encoder"])
def test_predictor_over_the_cache_matches_the_arena(arena, style, statements, kw):
    m = module(style=style, freeze=False, **kw)
    cache = D.EncoderCache(m, arena)
    res = []
    for src in (arena, cache):
        pr = D.FusedPredictor(m, capacity=400, statements=statements, top_k=5)
        for ids in id_lists(arena, 7, 29):
            pr.predict_ids(src, ids)
        res.append({k: v.clone() for k, v in pr.results().items()})
    assert set(res[0]) == set(res[1]) and ("embedding" in res[0]) == bool(kw)
    for k in res[0]:
        assert torch.equal(res[0][k].view(torch.int32), res[1][k].view(torch.int32)), k     # NaN past the last statement: bits


# ---- 6. stale captured graphs --------------------------------------------------------------------------------------------------
def test_a_changed_encoder_is_refused_instead_of_replayed(arena):
    m = module()
    tr = D.FusedTrainer(m, use_cuda_graph=True)
    ev = D.FusedEvaluator(m)
    cache = D.EncoderCache(m, arena)
    ids = [3, 1, 4, 1, 5]
    for _ in range(3):                               # eager, capture, replay
        tr.step_ids(cache, ids)
        ev.update_ids(cache, ids)
    assert tr._stream_slots[next(iter(tr._stream_slots))]["graph"] is not None
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    sd["ggnn.gru.weight_hh"].mul_(0.5)
    m.load_state_dict(sd)                            # in place, into the trainer's flat buffer
    with pytest.raises(ValueError, match="rebuild the cache"):
        tr.step_ids(cache, ids)
    with pytest.raises(ValueError, match="rebuild the cache"):
        ev.update_ids(cache, ids)
    fresh = D.EncoderCache(m, arena)
    tr.step_ids(fresh, ids)                          # a rebuilt cache trains on
    ev.update_ids(fresh, ids)
    torch.cuda.synchronize()
    assert not torch.equal(fresh.h, cache.h)


# ---- 7. a stale cache is released ----------------------------------------------------------------------------------------------
def _owner(kind, m):
    if kind == "trainer":
        tr = D.FusedTrainer(m, use_cuda_graph=True, max_graph_shapes=1)
        return tr, tr.step_ids
    if kind == "evaluator":
        ev = D.FusedEvaluator(m, max_graph_shapes=1)
        return ev, ev.update_ids
    pr = D.FusedPredictor(m, capacity=1000, max_graph_shapes=1)
    return pr, pr.predict_ids


@pytest.mark.parametrize("refused_first", [True, False], ids=["after-refusal", "on-rebuild"])
@pytest.mark.parametrize("kind", ["trainer", "evaluator", "predictor"])
def test_a_rebuilt_cache_frees_the_old_one(arena, kind, refused_first):
    """One owner across a checkpoint change: the old cache's slots go — when the old cache is refused, or when the rebuilt one
    makes its first slot — so the old planes are freed once the caller drops the cache, and the rebuilt cache is captured within
    max_graph_shapes = 1."""
    import gc
    import weakref
    m = module()
    owner, run = _owner(kind, m)
    ids = [2, 7, 1, 8]
    cache = D.EncoderCache(m, arena)
    for _ in range(3):                                   # eager, capture, replay
        run(cache, ids)
    torch.cuda.synchronize()
    old, nbytes = weakref.ref(cache), cache.nbytes
    base = torch.cuda.memory_allocated()                 # the old cache and its slot
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    sd["ggnn.gru.weight_ih"].mul_(0.5)
    m.load_state_dict(sd)
    if refused_first:
        with pytest.raises(ValueError, match="rebuild the cache"):
            run(cache, ids)
    del cache
    gc.collect()
    fresh = D.EncoderCache(m, arena)
    for _ in range(3):
        run(fresh, ids)
    torch.cuda.synchronize()
    gc.collect()
    assert old() is None, "the owner still holds the stale cache"
    grown = torch.cuda.memory_allocated() - base        # the fresh cache and its slot in place of the old ones: about 0
    assert grown < nbytes // 2, (grown, nbytes)
    (key, slot), = owner._stream_slots.items()
    assert key[:2] == ("cache", id(fresh)) and slot["graph"] is not None


# ---- 8. two ranks (NCCL) ---------------------------------------------------------------------------------------------------------
def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dp_worker(rank, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2", DDFA_DETERMINISTIC="1")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    try:
        big = synth.make_batch(80, 40, seed=31, variable=True, vuln_rate=0.3)
        arena = D.GraphArena.from_graphs([big], dev)
        rng = np.random.default_rng(40)
        shards = [[rng.choice(80, 12, replace=False) for _ in range(2)] for _ in range(5)]     # per step: the ids of rank 0 and 1
        out = {}
        for style, kw in (("graph", {}), ("node", {"undersample_node_on_loss_factor": 1.0})):
            runs = []
            for source in ("arena", "cache"):
                torch.manual_seed(3)
                m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, label_style=style, concat_all_absdf=True, positive_weight=2.0,
                                        engine="tcgen05", **kw).to(dev)
                for name, p in m.named_parameters():
                    if not name.startswith(("output_layer.", "pooling.")):
                        p.requires_grad_(False)
                tr = D.FusedTrainer(m, use_cuda_graph=True, distributed=True, exchange="auto", node_sample_seed=9)
                src = arena if source == "arena" else D.EncoderCache(m, arena)
                losses = []
                for step in shards + shards:             # twice: the second pass replays the captured steps
                    losses.append(float(tr.step_ids(src, step[rank], global_batch=24)))
                runs.append((losses, tr.flat_p.cpu(), tr.exp_avg.cpu(), tr.exp_avg_sq.cpu(), tr.exchange))
            (la, pa, ma, va, ex), (lc, pc, mc, vc, _) = runs
            out[style] = (ex, la == lc, bool(torch.equal(pa, pc) and torch.equal(ma, mc) and torch.equal(va, vc)), la)
        q.put((rank, out))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


def test_two_ranks_nccl_over_a_cache_match_the_arena():
    """Graph style (the small-gradient all-reduce overlapped with the backward) and node style (the loss rows drawn over the
    global batch) over NCCL: step_ids(cache) equals step_ids(arena) on every rank, bit for bit in deterministic mode."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(2):
            rank, out = q.get(timeout=600)
            res[rank] = out
    finally:
        for p in procs:
            p.join(timeout=120)
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(timeout=30)
    for r in (0, 1):
        assert not isinstance(res[r], str), res[r]
        for style in ("graph", "node"):
            exchange, same_loss, same_state, losses = res[r][style]
            assert exchange == "nccl" and same_loss and same_state, (r, style, losses)
