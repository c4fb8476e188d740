"""The batch paths of :class:`~deepdfa_b200.trainer.FusedTrainer` and :class:`~deepdfa_b200.evaluator.FusedEvaluator`: host
batches through static per-shape buffers, graph ids of an arena assembled inside the captured graph, resident device batches
with one captured graph each, and eager launches.
"""
from __future__ import annotations

import torch

from . import _lib
from . import engine as E
from .batched_graph import BatchedCFG, as_batched_cfg
from .encoder_cache import EncoderCache


def graph_step(device, graph, warm: bool, enqueue):
    """One step through a cached CUDA graph: ``enqueue()`` runs eagerly while the shape is not ``warm`` (its first visit grows
    the workspace and loads modules outside any capture); after that ``graph`` is replayed, captured first, after a device
    synchronise, when it is None.  Returns the graph (None when the step ran eagerly)."""
    if not warm:
        enqueue()
        return None
    if graph is None:
        torch.cuda.synchronize(device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            enqueue()
    graph.replay()
    return graph


def bucket_shape(N: int, Eg: int, bucket_nodes: int, bucket_edges: int, min_pad_nodes: int):
    """Padded (nodes, edges) of a batch under shape bucketing, or None when bucketing is off (``bucket_nodes <= 0``)."""
    if bucket_nodes <= 0:
        return None
    bn, be = bucket_nodes, max(bucket_edges, 1)
    Nb = (N + max(min_pad_nodes, 1) + bn - 1) // bn * bn
    Eb = (Eg + be - 1) // be * be
    return Nb, Eb


def new_stream_slot(g, bucket, device, valid_nodes_word: bool) -> dict:
    """The static per-shape input buffers of host batches shaped like ``g`` (or padded to ``bucket``): two buffer sets, so
    that while the graph of one set runs the next batch is copied into the other (prefetch).  ``valid_nodes_word``: every set
    gets an int32 device word with the batch's valid node count (node style under bucketing)."""
    src, dst = g.edges()
    N, Eg, B = g.num_nodes(), g.num_edges(), g.batch_size
    Ns, Es, Bs = (bucket[0], bucket[1], B + 1) if bucket else (N, Eg, B)

    def new_set():
        return {"src": torch.empty(Es, dtype=src.dtype, device=device), "dst": torch.empty(Es, dtype=dst.dtype, device=device),
                "bnn": torch.empty(Bs, dtype=torch.int64, device=device),
                "ndata": {k: torch.zeros((Ns,) + tuple(v.shape[1:]), dtype=v.dtype, device=device) for k, v in g.ndata.items()},
                "graph": None, "keep": None, "free": None, "ready": None, "result": None,
                "valid_nodes": torch.zeros(1, dtype=torch.int32, device=device) if (bucket and valid_nodes_word) else None}
    return {"sets": [new_set(), new_set()], "next": 0, "staged": None, "warm": False, "N": Ns,
            "valid": B if bucket else None,
            "iota": torch.arange(Es, dtype=src.dtype, device=device) if bucket else None}


def stage(slot, g, stream) -> int:
    """Copies the host batch ``g`` into the slot's next buffer set on ``stream``; returns the set index.  Under bucketing
    the tails are (re)written too: padding nodes get feature index 0 / _VULN 0, the padding edges become self loops spread
    round-robin over the padding nodes, and the dummy graph's node count goes into the last ``batch_num_nodes`` entry."""
    i = slot["next"]
    slot["next"] = 1 - i
    st = slot["sets"][i]
    caller = torch.cuda.current_stream()
    with torch.cuda.stream(stream):
        if st["free"] is not None:
            stream.wait_event(st["free"])           # the graph that last read this set has finished
        else:
            stream.wait_stream(caller)              # first use: the set's zero fill, enqueued on the caller's stream, is done
        src, dst = g.edges()
        N, Eg, B = g.num_nodes(), g.num_edges(), g.batch_size
        st["src"][:Eg].copy_(src, non_blocking=True)
        st["dst"][:Eg].copy_(dst, non_blocking=True)
        st["bnn"][:B].copy_(g.batch_num_nodes(), non_blocking=True)
        for k, v in g.ndata.items():
            st["ndata"][k][:N].copy_(v, non_blocking=True)
        if st["valid_nodes"] is not None:
            st["valid_nodes"].fill_(N)              # node style: the sampler leaves the padding nodes (the tail) out
        if slot["valid"] is not None:
            Nb, Eb = slot["N"], st["src"].shape[0]
            pad_nodes = Nb - N
            st["bnn"][B:].fill_(pad_nodes)
            for k in st["ndata"]:
                st["ndata"][k][N:].zero_()
            if Eb > Eg:
                torch.remainder(slot["iota"][: Eb - Eg], pad_nodes, out=st["src"][Eg:])
                st["src"][Eg:].add_(N)
                st["dst"][Eg:].copy_(st["src"][Eg:])
        ev = torch.cuda.Event()
        ev.record(stream)
        st["ready"] = ev
    return i


def arena_ids(arena, ids, who: str):
    """``(ids as int64 numpy, B, N, E)`` of the graph ids of ``arena``; raises IndexError for an empty list or a bad id."""
    import numpy as np
    ids_np = np.asarray(ids.cpu() if isinstance(ids, torch.Tensor) else ids, dtype=np.int64).reshape(-1)
    if ids_np.size == 0 or ids_np.min() < 0 or ids_np.max() >= arena.num_graphs:
        raise IndexError(f"{who}: empty id list or graph id out of range")
    return ids_np, int(ids_np.shape[0]), int(arena.nodes_per_graph[ids_np].sum()), int(arena.edges_per_graph[ids_np].sum())


def new_arena_slot(arena, B: int, N: int, Eg: int) -> dict:
    """Static per-shape outputs of the arena batch producer and a ring of pinned id stages: the host may run several steps
    ahead of the device (that is what the captured graph is for), so a stage is rewritten only after the H2D copy that last
    read it has completed."""
    return {"out": arena.alloc_outputs(B, N, Eg), "stages": [torch.empty(B, dtype=torch.int32).pin_memory() for _ in range(4)],
            "stage_done": [None] * 4, "turn": 0, "steps": 0,
            "graph": None, "warm": False, "keep": None, "arena": arena}     # the arena stays alive with its graph


def push_ids(slot, ids_np) -> None:
    """Copies the id list into the slot's next pinned stage and from there, in stream order, into its device id buffer; every
    256 calls the producer's device error counter of the last batch is checked (one synchronisation)."""
    import numpy as np
    k = slot["turn"]
    slot["turn"] = (k + 1) % len(slot["stages"])
    if slot["stage_done"][k] is not None:
        slot["stage_done"][k].synchronize()
    slot["stages"][k].copy_(torch.from_numpy(ids_np.astype(np.int32)))
    slot["out"]["ids"].copy_(slot["stages"][k], non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    slot["stage_done"][k] = ev
    slot["steps"] += 1
    if slot["keep"] is not None and slot["steps"] % 256 == 0:
        slot["keep"][0].check()      # the assembler's device error counter (bad id / totals mismatch): one sync every 256 steps


def new_cache_slot(cache, B: int, N: int) -> dict:
    """An arena slot's counterpart for an :class:`~deepdfa_b200.encoder_cache.EncoderCache`: the static outputs of
    ``ddfa_cache_batch`` and the same ring of pinned id stages."""
    return {"out": cache.alloc_outputs(B, N), "stages": [torch.empty(B, dtype=torch.int32).pin_memory() for _ in range(4)],
            "stage_done": [None] * 4, "turn": 0, "steps": 0,
            "graph": None, "warm": False, "keep": None, "arena": cache}     # the cache stays alive with its graph


def cache_graph(cb) -> E.DeviceGraph:
    """The :class:`~deepdfa_b200.engine.DeviceGraph` of a batch gathered from an encoder cache: graph_ptr only (no CSR; what
    runs after the GGNN reads none)."""
    return E.DeviceGraph(cb.num_nodes(), 0, cb.batch_size, None, None, None, None, cb.graph_ptr, cb.device)


class CapturedBatches:
    """The three batch paths, their caches and their capture policy, for a class that runs one batch at a time.

    The owner sets ``device``, ``_node`` (label_style="node") and the settings below, which are read when a batch runs, so they
    may change between batches: ``use_cuda_graph``, ``bucket_nodes`` / ``bucket_edges`` / ``bucket_min_pad_nodes`` (host
    batches), ``max_graph_shapes`` (host and arena slots kept; further shapes run eagerly) and ``max_resident_graphs``
    (resident batch objects captured; further ones run eagerly).  Its public methods pass a ``ctx`` through to its hooks:

    * ``_prepare(batch)``: ``(g, dg, ...)``, the ``BatchedCFG`` and the device graph first;
    * ``_key_suffix(ctx, B)``: what else, beyond shape, ``B`` and the deterministic mode, a captured graph bakes in;
    * ``_enqueue(ctx, prepared, vuln, num_valid, valid_nodes)``: the batch's launches, ``vuln`` its labels as contiguous int32
      on the device, ``num_valid`` the real graph count under bucketing (None: every graph is real), ``valid_nodes`` the int32
      device word of the real node count in node style under bucketing (None: every node is real).  What it returns is kept
      with the captured graph;
    * ``_after_run(result, num_nodes)``: after every run, replays included, with that result and the batch's real node count;
    * ``_check_cache(cache, who)`` and ``_prepare_cache(cb)``: the id path over an encoder cache (``_run_ids`` with an
      :class:`~deepdfa_b200.encoder_cache.EncoderCache`): what the owner refuses to run from cached rows (it raises), and the
      ``prepared`` tuple of a gathered batch, whose device graph has graph_ptr only and whose embedding indices are the
      :class:`~deepdfa_b200.encoder_cache.CachedRows`.

    ``_stream_slots`` (host and arena slots) and ``_graphs`` (resident graphs, the graph at index 0 of each entry) are the live
    caches: clearing them drops the captured graphs."""

    def __init__(self):
        self._stream_slots = {}
        self._graphs = {}
        self._warm_shapes = set()
        self._copy_stream = None

    def _key_suffix(self, ctx, B: int) -> tuple:
        return ()

    def _vuln(self, g) -> torch.Tensor:
        """The batch's ``_VULN`` as contiguous int32 on the device; a converted copy is cached on the graph object."""
        vuln = g.ndata["_VULN"]
        if vuln.device != self.device or vuln.dtype != torch.int32 or not vuln.is_contiguous():
            cached = g._cache.get("vuln_dev")
            if cached is None:
                cached = vuln.to(self.device, non_blocking=True).to(torch.int32).contiguous()
                g._cache["vuln_dev"] = cached
            vuln = cached
        return vuln

    def _drop_graphs(self) -> None:
        """Forgets every captured graph (host sets, arena slots, resident batches); the next visits capture anew."""
        for slot in self._stream_slots.values():
            for st in slot.get("sets", [slot]):
                st["graph"] = None
        self._graphs.clear()

    def _run(self, batch, ctx) -> None:
        g = as_batched_cfg(batch) if self.use_cuda_graph else None
        if g is not None and g.device.type == "cpu":
            self._run_host(batch, g, ctx)
        else:
            self._run_resident(batch, ctx)

    # ---- host batches through per-shape static buffers ---------------------------------------------------------------------
    def _host_slot(self, g, ctx):
        N, Eg, B = g.num_nodes(), g.num_edges(), g.batch_size
        bucket = bucket_shape(N, Eg, self.bucket_nodes, self.bucket_edges, self.bucket_min_pad_nodes)
        # keyed by the deterministic mode too: a captured graph keeps the kernels of the mode it was captured in
        det = _lib.deterministic_requested()
        key = ("bucket", bucket[0], bucket[1], B, det) if bucket else ("exact", N, Eg, B, det)
        key += self._key_suffix(ctx, B)
        slot = self._stream_slots.get(key)
        if slot is None:
            if len(self._stream_slots) >= self.max_graph_shapes:
                return None
            slot = new_stream_slot(g, bucket, self.device, self._node)
            self._stream_slots[key] = slot
        return slot

    def _prefetch(self, batch, ctx) -> None:
        if not self.use_cuda_graph:
            return
        g = as_batched_cfg(batch)
        if g.device.type != "cpu":
            return
        with torch.cuda.device(self.device):
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream(device=self.device)
            slot = self._host_slot(g, ctx)
            if slot is not None:
                slot["staged"] = (id(batch), stage(slot, g, self._copy_stream))

    def _run_host(self, batch, g, ctx) -> None:
        """Host batch + use_cuda_graph: the batch's arrays are copied into device buffers that are STATIC per shape
        (num_nodes, num_edges, batch_size — or per BUCKET shape with ``bucket_nodes`` / ``bucket_edges``) and one captured
        CUDA graph per buffer set covers the whole batch including the device CSR build — a new batch of a known shape costs
        its H2D copies (overlappable: ``prefetch``) plus one graph launch.  The first visit of a shape runs eagerly
        (workspace growth), the next two capture."""
        with torch.cuda.device(self.device):
            slot = self._host_slot(g, ctx)
            if slot is None:          # more shapes than max_graph_shapes: same kernels, launched eagerly
                return self._run_resident(batch, ctx)
            N = slot["N"]
            main = torch.cuda.current_stream()
            staged = slot["staged"]
            slot["staged"] = None
            if staged is not None and staged[0] == id(batch):
                i = staged[1]
                main.wait_event(slot["sets"][i]["ready"])
            else:
                i = stage(slot, g, main)
            st = slot["sets"][i]

            def enqueue():
                gs = BatchedCFG(st["src"], st["dst"], st["bnn"], dict(st["ndata"]), num_nodes=N)   # no cached device CSR
                prepared = self._prepare(gs)
                vuln = self._vuln(gs)
                st["result"] = self._enqueue(ctx, prepared, vuln, slot["valid"], st["valid_nodes"])
                st["keep"] = prepared + (vuln,)         # tensors allocated during capture live in the graph's pool

            st["graph"] = graph_step(self.device, st["graph"], slot["warm"], enqueue)
            slot["warm"] = True
            self._after_run(st["result"], g.num_nodes())
            ev = torch.cuda.Event()
            ev.record(main)
            st["free"] = ev

    # ---- graph ids of an arena, assembled inside the captured graph ----------------------------------------------------------
    def _run_ids(self, arena, ids, ctx, who: str) -> None:
        if isinstance(arena, EncoderCache):
            return self._run_cache(arena, ids, ctx, who)
        if not self.use_cuda_graph:
            return self._run_resident(arena.batch(ids), ctx)
        ids_np, B, N, Eg = arena_ids(arena, ids, who)
        key = ("arena", id(arena), N, Eg, B, _lib.deterministic_requested()) + self._key_suffix(ctx, B)
        slot = self._stream_slots.get(key)
        with torch.cuda.device(self.device):
            if slot is None:
                if len(self._stream_slots) >= self.max_graph_shapes:
                    return self._run_resident(arena.batch(ids), ctx)
                slot = new_arena_slot(arena, B, N, Eg)
                self._stream_slots[key] = slot
            push_ids(slot, ids_np)

            def enqueue():
                g = arena._assemble(slot["out"]["ids"], B, N, Eg, slot["out"])
                prepared = self._prepare(g)
                vuln = self._vuln(g)
                slot["result"] = self._enqueue(ctx, prepared, vuln, None, None)
                slot["keep"] = prepared + (vuln,)       # keep[0]: the assembled batch, whose error counter push_ids checks

            slot["graph"] = graph_step(self.device, slot["graph"], slot["warm"], enqueue)
            slot["warm"] = True
            self._after_run(slot["result"], N)

    def _run_cache(self, cache, ids, ctx, who: str) -> None:
        """Graph ids over an encoder cache: the batch's rows, labels and graph_ptr gathered by ``ddfa_cache_batch`` into static
        per-shape buffers inside the captured graph, then the owner's launches after the GGNN.  The cache is checked against the
        module first, so a stale captured graph is never replayed; a cache that fails the check loses its slots, and so does,
        when a new slot is made, every other cache that no longer matches the module.  Beyond ``max_graph_shapes`` slots, or without
        ``use_cuda_graph``, the same launches run eagerly over freshly allocated outputs."""
        self._check_cache(cache, who)
        try:
            cache.check(self.module)
        except ValueError:
            self._drop_cache_slots(lambda c: c is cache)      # its graphs can never replay again: free them and the cache
            raise
        ids_np, B, N, _ = arena_ids(cache.arena, ids, who)
        key = ("cache", id(cache), N, B, _lib.deterministic_requested()) + self._key_suffix(ctx, B)
        with torch.cuda.device(self.device):
            slot = self._stream_slots.get(key) if self.use_cuda_graph else None
            if slot is None and self.use_cuda_graph:
                # slots of caches that no longer match the module (a rebuilt cache's predecessor) hold the old planes and
                # count against max_graph_shapes: they go before a new slot is counted
                self._drop_cache_slots(lambda c: c is not cache and not c.matches(self.module))
                if len(self._stream_slots) < self.max_graph_shapes:
                    slot = new_cache_slot(cache, B, N)
                    self._stream_slots[key] = slot
            if slot is None:
                cb = cache.batch(ids_np)
                self._after_run(self._enqueue(ctx, self._prepare_cache(cb), self._vuln(cb), None, None), N)
                return
            push_ids(slot, ids_np)

            def enqueue():
                cb = cache._assemble(slot["out"]["ids"], B, N, slot["out"])
                prepared = self._prepare_cache(cb)
                vuln = self._vuln(cb)
                slot["result"] = self._enqueue(ctx, prepared, vuln, None, None)
                slot["keep"] = prepared + (vuln,)       # keep[0]: the gathered batch, whose error counter push_ids checks

            slot["graph"] = graph_step(self.device, slot["graph"], slot["warm"], enqueue)
            slot["warm"] = True
            self._after_run(slot["result"], N)

    def _drop_cache_slots(self, stale) -> None:
        """Forgets the slots (static outputs, captured graph, id stages) of every encoder cache ``c`` with ``stale(c)``, and with
        them this owner's references to those caches, so a cache nothing else holds is freed.  Waits for the device first when
        a captured graph is among them: it may still be running."""
        keys = [k for k, s in self._stream_slots.items() if k[0] == "cache" and stale(s["arena"])]
        if any(self._stream_slots[k]["graph"] is not None for k in keys):
            torch.cuda.synchronize(self.device)
        for k in keys:
            del self._stream_slots[k]

    # ---- device-resident batch objects, or eager launches --------------------------------------------------------------------
    def _run_resident(self, batch, ctx) -> None:
        """One captured CUDA graph per resident batch object when ``use_cuda_graph`` (its device pointers are baked in), once
        its shape has run eagerly; a batch that cannot be captured runs eagerly."""
        prepared = self._prepare(batch)
        g, dg = prepared[0], prepared[1]
        vuln = self._vuln(g)
        suffix = self._key_suffix(ctx, dg.batch_size)
        with torch.cuda.device(self.device):
            det = _lib.deterministic_requested()
            shape_key = (dg.num_nodes, dg.num_edges, dg.batch_size, det) + suffix
            graph_key = (id(g), det) + suffix
            capturable = self.use_cuda_graph and g.device.type == "cuda" and \
                (graph_key in self._graphs or len(self._graphs) < self.max_resident_graphs)
            entry = self._graphs.get(graph_key)
            out = {}

            def enqueue():
                out["result"] = self._enqueue(ctx, prepared, vuln, None, None)
            cg = graph_step(self.device, entry[0] if entry else None, capturable and shape_key in self._warm_shapes, enqueue)
            if entry is None and cg is not None:
                self._graphs[graph_key] = (cg, prepared, vuln, out["result"])     # keep the captured tensors alive
            self._warm_shapes.add(shape_key)
            self._after_run(out["result"] if "result" in out else entry[3], dg.num_nodes)
