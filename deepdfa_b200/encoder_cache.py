"""Device-resident cache of a frozen graph encoder's output over a whole :class:`~deepdfa_b200.arena.GraphArena`.

With the embedding tables and the GatedGraphConv frozen (the reference's ``--freeze_graph ckpt``, main_cli.py:136-144), what the
readout, the node head and their backward read of the GGNN is, per node, ``h_T`` and ``x`` (the embedding rows), and neither can
change between epochs.  :class:`EncoderCache` computes both once, for every node of the arena, and keeps them on the device:

    cache = EncoderCache(model, arena)              # one inference-form GGNN pass over the arena
    trainer.step_ids(cache, ids)                    # ddfa_cache_batch + readout / head, loss, head backward, Adam
    evaluator.update_ids(cache, ids); predictor.predict_ids(cache, ids)

A batch is then a gather of its graphs' rows (``ddfa_cache_batch``): no CSR, no embedding, no GGNN launch.

Footprint: ``2 * N_all * D * 4`` bytes (two fp32 planes) — about 10.6 GB for Big-Vul's 10.4 M nodes at D = 128.

Invalidation: the cache records the ``data_ptr()`` and ``_version`` of the K embedding tables and of the six GatedGraphConv
tensors, the engine and the deterministic mode it was built under; :meth:`EncoderCache.check` raises ``ValueError`` once any of
them differs (``load_state_dict`` into the module bumps ``_version``; a ``FusedTrainer`` built after the cache moves the
parameters into its flat buffer, a new ``data_ptr``).  Writes that bypass the version counter — ``p.data.copy_(...)``, or an
optimizer updating the encoder through raw pointers — are not seen: the cache is for an encoder that stays frozen.
"""
from __future__ import annotations

import weakref
import numpy as np
import torch

from . import _lib
from . import engine as E
from .module import _ENGINES

# the fingerprinted tensors of ``module.param_list()``: the K tables, then these six
_GGNN_NAMES = ("ggnn.linears.0.weight", "ggnn.linears.0.bias", "ggnn.gru.weight_ih", "ggnn.gru.weight_hh", "ggnn.gru.bias_ih",
               "ggnn.gru.bias_hh")


class CachedRows:
    """The GGNN outputs of a batch taken from an encoder cache, ``x`` (embedding rows) and ``h`` (h_T), [N, D] each: what a
    batch prepared from a cache carries where a prepared graph batch carries its embedding indices."""

    __slots__ = ("x", "h")

    def __init__(self, x: torch.Tensor, h: torch.Tensor):
        self.x, self.h = x, h


class CacheBatch:
    """A batch gathered from an :class:`EncoderCache` by ``ddfa_cache_batch``: ``graph_ptr``, ``_VULN`` (``ndata``) and the
    rows (``rows``).  It has no edges: only what the readout, the node head and their backward read."""

    def __init__(self, graph_ptr: torch.Tensor, vuln: torch.Tensor, rows: CachedRows, ws: torch.Tensor, num_nodes: int):
        self.graph_ptr = graph_ptr
        self.ndata = {"_VULN": vuln}
        self.rows = rows
        self.batch_size = graph_ptr.numel() - 1
        self._n = int(num_nodes)
        self._ws = ws                       # [error counter int32][node_ptr int32[B+1]]
        self._cache = {}
        self.device = graph_ptr.device

    def num_nodes(self) -> int:
        return self._n

    def check(self) -> None:
        """Synchronising check of the assembler's error counter (bad graph id / node total mismatch)."""
        err = int(self._ws.view(torch.int32)[0].item())
        if err:
            raise _lib.DdfaError(f"cache batch: {err & 0xffff} graph id(s) out of range, totals mismatch={bool(err >> 16)}")


def _encoder_tensors(model):
    return model.param_list()[:len(model._tables()) + 6]


def encoder_names(model):
    """The names of the fingerprinted tensors, in ``_encoder_tensors`` order."""
    names = {id(p): n for n, p in model.named_parameters()}
    return [names.get(id(t), n) for t, n in zip(_encoder_tensors(model), [f"table{i}" for i in range(len(model._tables()))]
                                                 + list(_GGNN_NAMES))]


def _fingerprint(model):
    return tuple((t.data_ptr(), t._version) for t in _encoder_tensors(model))


class EncoderCache:
    def __init__(self, model, arena, graphs_per_batch: int = 1024):
        """Runs ``model``'s GGNN forward (embedding + T GatedGraphConv steps, the inference form ``engine.forward(training=False,
        head=False)``: the kernels a frozen-encoder ``FusedTrainer`` step runs) over every graph of ``arena`` and keeps
        ``h`` (h_T) and ``x`` (the embedding rows), fp32 ``[N_all, D]`` each, in arena node order.  The pass runs over
        contiguous id ranges of ``graphs_per_batch`` graphs (which bound its workspace), each range's rows landing in a
        contiguous slice of the planes.  Raises ``IndexError`` when a node feature index lies outside the embedding tables."""
        if model.device.type != "cuda" or arena.device != model.device:
            raise _lib.DdfaError("EncoderCache needs the module and the arena on the same CUDA device (no CPU fallback)")
        gpb = int(graphs_per_batch)
        if gpb < 1:
            raise ValueError(f"graphs_per_batch must be >= 1, got {graphs_per_batch!r}")
        self.arena = arena
        self.device = arena.device
        self._record(model)
        K = len(model._tables())
        self.D = K * model._tables()[0].shape[1]
        self.num_nodes = int(arena.vuln.numel())
        G = arena.num_graphs
        node_off = np.concatenate([[0], np.cumsum(arena.nodes_per_graph)]).astype(np.int64)
        params = E.ParamPack.from_flat_list([p.data for p in model.param_list()], K, model._num_layers)
        eng, T = _ENGINES[model.engine], model.hparams.n_steps
        dev = self.device
        with torch.cuda.device(dev):
            self.h = torch.empty(self.num_nodes, self.D, dtype=torch.float32, device=dev)
            self.x = torch.empty(self.num_nodes, self.D, dtype=torch.float32, device=dev)
            oob = torch.zeros(1, dtype=torch.int32, device=dev)
            ws = E.Workspace(dev)
            for lo in range(0, G, gpb):
                hi = min(G, lo + gpb)
                n_lo, n_hi = int(node_off[lo]), int(node_off[hi])
                if n_hi == n_lo:
                    continue                        # only 0-node graphs: no row to compute
                b = arena.batch(np.arange(lo, hi))
                dg = E.prepare_graph(b, dev)        # the CSR ddfa_arena_batch attached
                idx = E.node_indices(b, model.concat_all_absdf, model.feature_keys["feature"], dev)
                x, h, _ = E.forward(params, dg, idx, T, training=False, engine=eng, alloc=ws, head=False, oob_counter=oob)
                self.x[n_lo:n_hi].copy_(x)
                self.h[n_lo:n_hi].copy_(h)
            bad = int(oob.item())
        if bad:
            raise IndexError(f"EncoderCache: {bad} node feature indices outside [0, {model.input_dim}) in the arena")

    def _record(self, model) -> None:
        """The fingerprint :meth:`check` compares against: the module, its engine, the deterministic mode, and (data_ptr,
        _version) of every table and GatedGraphConv tensor."""
        self.engine = model.engine
        self.deterministic = _lib.deterministic_requested()
        self._module = weakref.ref(model)
        self._fp = _fingerprint(model)

    @property
    def num_graphs(self) -> int:
        return self.arena.num_graphs

    @property
    def nbytes(self) -> int:
        """Bytes of the two planes: ``2 * N_all * D * 4``."""
        return 2 * self.num_nodes * self.D * 4

    def check(self, model) -> None:
        """Raises ``ValueError`` when ``model`` is not the module the cache was built from, or when its encoder no longer
        matches what the cache holds: a table or GatedGraphConv tensor with another ``data_ptr()`` or ``_version``, another
        engine, or another deterministic mode than at build time.  The message says to rebuild the cache."""
        if self._module() is not model:
            raise ValueError("EncoderCache: the cache was built from another module; build an EncoderCache of this one")
        if model.engine != self.engine:
            raise ValueError(f"EncoderCache: built under engine={self.engine!r}, the module now runs {model.engine!r}: rebuild the cache")
        det = _lib.deterministic_requested()
        if det != self.deterministic:
            raise ValueError(f"EncoderCache: built with deterministic mode {'on' if self.deterministic else 'off'}, it is now "
                             f"{'on' if det else 'off'}: rebuild the cache")
        fp = _fingerprint(model)
        if fp != self._fp:
            changed = [n for n, a, b in zip(encoder_names(model), fp, self._fp) if a != b]
            raise ValueError(f"EncoderCache: the encoder changed since the cache was built ({', '.join(changed)}: new storage or "
                             "an in-place write): rebuild the cache")

    def matches(self, model) -> bool:
        """Whether :meth:`check` passes for ``model``."""
        try:
            self.check(model)
        except ValueError:
            return False
        return True

    # ---- batch assembly (ddfa_cache_batch) -------------------------------------------------------------------------------------
    def batch(self, ids) -> CacheBatch:
        """The rows, labels and graph_ptr of the graphs ``ids`` (host sequence / numpy / CPU tensor, repeats allowed) in that
        order, in freshly allocated outputs."""
        ids_np = np.asarray(ids.cpu() if isinstance(ids, torch.Tensor) else ids, dtype=np.int64).reshape(-1)
        if ids_np.size == 0 or ids_np.min() < 0 or ids_np.max() >= self.num_graphs:
            raise IndexError("EncoderCache.batch: empty id list or graph id out of range")
        B, N = int(ids_np.shape[0]), int(self.arena.nodes_per_graph[ids_np].sum())
        with torch.cuda.device(self.device):
            o = self.alloc_outputs(B, N)
            o["ids"].copy_(torch.from_numpy(ids_np.astype(np.int32)), non_blocking=True)
            return self._assemble(o["ids"], B, N, o)

    def alloc_outputs(self, B: int, N: int) -> dict:
        dev = self.device
        i32 = dict(dtype=torch.int32, device=dev)
        wsb = _lib.lib().call("ddfa_cache_batch_workspace_bytes", B)
        return {"ids": torch.empty(B, **i32), "graph_ptr": torch.empty(B + 1, **i32), "vuln": torch.empty(N, **i32),
                "h": torch.empty(N, self.D, dtype=torch.float32, device=dev), "x": torch.empty(N, self.D, dtype=torch.float32, device=dev),
                "ws": torch.empty(wsb, dtype=torch.uint8, device=dev)}

    def _assemble(self, ids_dev: torch.Tensor, B: int, N: int, o: dict) -> CacheBatch:
        a = self.arena
        _lib.lib().call("ddfa_cache_batch", E._p(ids_dev), B, a.num_graphs, E._p(a.node_off), E._p(a.vuln), E._p(self.h), E._p(self.x),
                        self.num_nodes, self.D, N, E._p(o["graph_ptr"]), E._p(o["vuln"]), E._p(o["h"]), E._p(o["x"]), E._p(o["ws"]),
                        o["ws"].numel(), E._stream_ptr())
        return CacheBatch(o["graph_ptr"], o["vuln"], CachedRows(o["x"], o["h"]), o["ws"], N)
