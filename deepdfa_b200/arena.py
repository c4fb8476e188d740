"""Device-resident graph arena + batch producer (SURVEY.md §8 row f1).

The reference assembles every training batch on the host: ``dgl.batch([...])`` inside the ``GraphDataLoader`` collate
(``DDFA/sastvd/linevd/datamodule.py:116-141``) or on the fly in ``BigVulDatasetLineVD.get_indices``
(``DDFA/sastvd/linevd/dataset.py:63-76`` — ``dgl.batch([self[i] for i in ...]).to(device)``), after which DGL builds its
CSR lazily on the device.  An 80 GB H100 holds the whole Big-Vul graph set (~10^7 nodes) many times over, so here the
dataset is uploaded ONCE — already in the layout the kernels read — and a batch is a list of graph ids:

    arena = GraphArena.from_graphs(list_of_single_graphs, device="cuda")     # one-time: H2D + one ddfa_build_csr
    batch = arena.batch(ids)            # device-side slice/rebase (ddfa_arena_batch), no host collate, no CSR build
    logits = model(batch, {}) ; loss = trainer.step(batch)

``arena.batch`` returns an :class:`ArenaBatch` — a :class:`BatchedCFG` (same ``ndata`` / ``batch_num_nodes`` / ``edges``
surface) whose device CSR is already attached, bit-identical to what ``prepare_graph(dgl.batch(graphs[ids]))`` builds.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from . import batched_graph as BG
from . import engine as E
from ._lib import DdfaError, ptr_array
from .batched_graph import BatchedCFG


class ArenaBatch(BatchedCFG):
    """A batch cut out of a :class:`GraphArena`.  The COO edge list (``edges()``) is materialised from the CSR on demand."""

    def __init__(self, dg: "E.DeviceGraph", bnn: torch.Tensor, ndata: Dict[str, torch.Tensor], ws: torch.Tensor):
        empty = torch.empty(0, dtype=torch.int64, device=dg.device)
        super().__init__(empty, empty, bnn, ndata, None, num_nodes=dg.num_nodes)
        self._dg = dg
        self._ws = ws                      # workspace of the producing call: [edge_ptr int32[B+1]][error counter int32][node_ptr int32[B+1]]
        self._coo = None
        self._cache[f"devgraph:{dg.device}:1"] = dg

    def num_edges(self) -> int:
        return self._dg.num_edges

    number_of_edges = num_edges

    @property
    def device(self) -> torch.device:
        return self._dg.device

    def edges(self):
        if self._coo is None:              # CSR by destination -> (src, dst), grouped by destination
            dg = self._dg
            deg = (dg.indptr[1:] - dg.indptr[:-1]).to(torch.int64)
            dst = torch.repeat_interleave(torch.arange(dg.num_nodes, device=dg.device, dtype=torch.int64), deg)
            self._coo = (dg.indices[: dg.num_edges].to(torch.int64), dst)
        return self._coo

    def batch_num_edges(self) -> torch.Tensor:
        ep = self._ws.view(torch.int32)[: self.batch_size + 1]
        return (ep[1:] - ep[:-1]).to(torch.int64)

    def check(self) -> None:
        """Synchronising check of the producer's error counter (bad graph id / inconsistent totals)."""
        err = int(self._ws.view(torch.int32)[self.batch_size + 1].item())
        if err:
            raise DdfaError(f"arena batch: {err & 0xffff} graph id(s) out of range, totals mismatch={bool(err >> 16)}")

    def to(self, device, non_blocking: bool = False):
        if torch.device(device) == self.device:
            return self
        src, dst = self.edges()
        return BatchedCFG(src, dst, self._bnn, self.ndata, None, num_nodes=self._n).to(device, non_blocking)

    def pin_memory(self):
        raise DdfaError("an ArenaBatch lives on the device")


class GraphArena:
    """All graphs of a dataset, resident on one GPU: CSR + transposed CSR over the disjoint union, node data, sizes."""

    def __init__(self, dg: "E.DeviceGraph", node_off: torch.Tensor, feats: Dict[str, torch.Tensor], vuln: torch.Tensor,
                 nodes_per_graph: np.ndarray, edges_per_graph: np.ndarray):
        self.dg = dg
        self.device = dg.device
        self.node_off = node_off                      # int32 [G+1] on the device
        self.feats = feats                            # name -> int64 [N_all] on the device (every ndata key except _VULN)
        self.vuln = vuln                              # int32 [N_all]
        self.nodes_per_graph = nodes_per_graph        # host copies: they size a batch without a device round trip
        self.edges_per_graph = edges_per_graph
        self._ids_stage: Optional[torch.Tensor] = None

    # ------------------------------------------------------------------------------------------------
    @classmethod
    def from_graphs(cls, graphs: Sequence, device="cuda") -> "GraphArena":
        """``graphs``: single graphs (or batches — their members become individual arena entries), DGL or BatchedCFG."""
        device = torch.device(device)
        singles: List[BatchedCFG] = []
        for g in graphs:
            g = BG.as_batched_cfg(g)
            singles.extend(BG.unbatch(g) if g.batch_size != 1 else [g])
        if not singles:
            raise ValueError("GraphArena.from_graphs: no graphs")
        return cls.from_union(BG.batch(singles), device)

    @classmethod
    def from_union(cls, big: BatchedCFG, device="cuda") -> "GraphArena":
        """The arena of ``big``, the disjoint union of its graphs as ``dgl.batch`` lays it out (COO with node ids offset per
        graph, ``batch_num_nodes`` / ``batch_num_edges``, ndata), on the host or already on ``device``.  Shared by
        :meth:`from_graphs` and :func:`deepdfa_b200.bigvul_io.load_arena`."""
        device = torch.device(device)
        if big.num_nodes() >= 2 ** 31 or big.num_edges() >= 2 ** 31:
            raise ValueError("GraphArena: more than 2^31 nodes or edges")
        if len([k for k in big.ndata if k != "_VULN"]) > 8:
            raise ValueError("GraphArena: at most 8 node-feature vectors")
        nodes = big.batch_num_nodes().cpu().numpy().astype(np.int64)
        edges = big.batch_num_edges().cpu().numpy().astype(np.int64)
        dg = E.prepare_graph(big.to(device), device, need_transpose=True)
        node_off = torch.zeros(len(nodes) + 1, dtype=torch.int32)
        node_off[1:] = torch.from_numpy(np.cumsum(nodes)).to(torch.int32)
        feats, vuln = {}, None
        for k, v in big.ndata.items():
            if k == "_VULN":
                vuln = v.to(device).to(torch.int32).contiguous()
            else:
                feats[k] = v.to(device).to(torch.int64).contiguous()
        if vuln is None:
            vuln = torch.zeros(big.num_nodes(), dtype=torch.int32, device=device)
        return cls(dg, node_off.to(device), feats, vuln, nodes, edges)

    @property
    def num_graphs(self) -> int:
        return int(self.nodes_per_graph.shape[0])

    # ------------------------------------------------------------------------------------------------
    def batch(self, ids, out: Optional[dict] = None) -> ArenaBatch:
        """Batch of the graphs ``ids`` (host sequence / numpy / CPU tensor, repeats allowed) in that order.  ``out``: optional
        dict of preallocated device tensors to write into (used by FusedTrainer's per-shape static buffers)."""
        ids_np = np.asarray(ids.cpu() if isinstance(ids, torch.Tensor) else ids, dtype=np.int64).reshape(-1)
        B = int(ids_np.shape[0])
        if B == 0:
            raise ValueError("GraphArena.batch: empty id list")
        if ids_np.min() < 0 or ids_np.max() >= self.num_graphs:
            raise IndexError("GraphArena.batch: graph id out of range")
        N = int(self.nodes_per_graph[ids_np].sum())
        Eg = int(self.edges_per_graph[ids_np].sum())
        dev = self.device
        L = _lib.lib()
        with torch.cuda.device(dev):
            ids_host = torch.from_numpy(ids_np.astype(np.int32))
            if out is not None:
                ids_dev = out["ids"]
                ids_dev.copy_(ids_host, non_blocking=True)
                return self._assemble(ids_dev, B, N, Eg, out)
            ids_dev = ids_host.to(dev, non_blocking=True)
            return self._assemble(ids_dev, B, N, Eg, self.alloc_outputs(B, N, Eg))

    def alloc_outputs(self, B: int, N: int, Eg: int) -> dict:
        dev = self.device
        i32 = dict(dtype=torch.int32, device=dev)
        wsb = _lib.lib().call("ddfa_arena_batch_workspace_bytes", B)
        return {"ids": torch.empty(B, **i32), "graph_ptr": torch.empty(B + 1, **i32), "indptr": torch.empty(N + 1, **i32),
                "indices": torch.empty(max(Eg, 1), **i32), "indptr_t": torch.empty(N + 1, **i32),
                "indices_t": torch.empty(max(Eg, 1), **i32), "vuln": torch.empty(N, **i32),
                "feats": {k: torch.empty(N, dtype=torch.int64, device=dev) for k in self.feats},
                "ws": torch.empty(wsb, dtype=torch.uint8, device=dev)}

    def _assemble(self, ids_dev: torch.Tensor, B: int, N: int, Eg: int, o: dict) -> ArenaBatch:
        L = _lib.lib()
        keys = list(self.feats)
        dg = self.dg
        L.call("ddfa_arena_batch", E._p(ids_dev), B, self.num_graphs, E._p(self.node_off), E._p(dg.indptr), E._p(dg.indices),
               E._p(dg.indptr_t), E._p(dg.indices_t), ptr_array([E._p(self.feats[k]) for k in keys]), len(keys), E._p(self.vuln), N, Eg,
               E._p(o["graph_ptr"]), E._p(o["indptr"]), E._p(o["indices"]), E._p(o["indptr_t"]), E._p(o["indices_t"]),
               ptr_array([E._p(o["feats"][k]) for k in keys]), E._p(o["vuln"]), E._p(o["ws"]), o["ws"].numel(), E._stream_ptr())
        bdg = E.DeviceGraph(N, Eg, B, o["indptr"], o["indices"], o["indptr_t"], o["indices_t"], o["graph_ptr"], self.device)
        bnn = (o["graph_ptr"][1:] - o["graph_ptr"][:-1]).to(torch.int64)
        ndata = dict(o["feats"])
        ndata["_VULN"] = o["vuln"]
        return ArenaBatch(bdg, bnn, ndata, o["ws"])
