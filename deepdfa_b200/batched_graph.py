"""Batched control-flow-graph container.

Duck-types the slice of ``dgl.DGLGraph`` that the DDFA hot path touches
(SURVEY.md Appendix C): ``ndata[...]`` (reference ``ggnn.py:87,91``;
``base_module.py:85``), ``batch_num_nodes()`` / ``batch_size`` (used by DGL's
``GlobalAttentionPooling`` called at ``ggnn.py:102`` and by
``base_module.py:87``), ``edges()`` (consumed by ``GatedGraphConv`` at
``ggnn.py:95``), ``num_nodes()``, ``num_edges()``, ``to()``, ``device``, plus
module-level ``batch`` / ``unbatch`` mirroring ``dgl.batch`` (``dataset.py:76``)
and ``dgl.unbatch`` (``base_module.py:87``).

Edge semantics are DGL's: a message flows ``src -> dst`` and is aggregated at
``dst``.  Node ids of a batch are contiguous per graph, as after ``dgl.batch``.

A real ``dgl.DGLGraph`` (when DGL is installed) is accepted everywhere a
``BatchedCFG`` is, through :func:`as_batched_cfg`.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence

import torch

ABS_DATAFLOW_SUBKEYS = ("api", "datatype", "literal", "operator")  # reference ggnn.py:17-19


class BatchedCFG:
    """A batch of homogeneous directed graphs with node data."""

    def __init__(self, src: torch.Tensor, dst: torch.Tensor, batch_num_nodes: torch.Tensor,
                 ndata: Optional[Dict[str, torch.Tensor]] = None,
                 batch_num_edges: Optional[torch.Tensor] = None, num_nodes: Optional[int] = None):
        if src.shape != dst.shape or src.dim() != 1:
            raise ValueError("src and dst must be 1-D tensors of equal length")
        self._src = src
        self._dst = dst
        self._bnn = batch_num_nodes.to(torch.int64)
        self._bne = batch_num_edges
        self.ndata: Dict[str, torch.Tensor] = dict(ndata or {})
        if num_nodes is not None:
            self._n = int(num_nodes)              # known by the caller: no reduction (and no device sync)
        elif self._bnn.is_cuda and self.ndata:
            self._n = int(next(iter(self.ndata.values())).shape[0])   # avoid a device reduction + sync
        else:
            self._n = int(self._bnn.sum().item()) if self._bnn.numel() else 0
        for k, v in self.ndata.items():
            if v.shape[0] != self._n:
                raise ValueError(f"ndata[{k!r}] has {v.shape[0]} rows, graph has {self._n} nodes")
        # device-side caches owned by the CUDA module (CSR/CSC); keyed by device
        self._cache: Dict[str, object] = {}

    # ---- DGLGraph subset -------------------------------------------------
    def edges(self):
        return self._src, self._dst

    def num_nodes(self) -> int:
        return self._n

    def num_edges(self) -> int:
        return int(self._src.shape[0])

    number_of_nodes = num_nodes
    number_of_edges = num_edges

    def batch_num_nodes(self) -> torch.Tensor:
        return self._bnn

    def batch_num_edges(self) -> torch.Tensor:
        if self._bne is None:
            # derive from dst ownership: nodes of graph b are [ptr[b], ptr[b+1])
            ptr = torch.zeros(self.batch_size + 1, dtype=torch.int64, device=self._bnn.device)
            ptr[1:] = torch.cumsum(self._bnn, 0)
            gid = torch.bucketize(self._dst.to(torch.int64), ptr[1:].to(self._dst.device), right=True)
            self._bne = torch.bincount(gid, minlength=self.batch_size).to(self._bnn.device)
        return self._bne

    @property
    def batch_size(self) -> int:
        return int(self._bnn.shape[0])

    @property
    def device(self) -> torch.device:
        return self._src.device

    @property
    def is_homogeneous(self) -> bool:
        return True

    def to(self, device, non_blocking: bool = False) -> "BatchedCFG":
        device = torch.device(device)
        if device == self.device:
            return self
        g = BatchedCFG(
            self._src.to(device, non_blocking=non_blocking),
            self._dst.to(device, non_blocking=non_blocking),
            self._bnn.to(device, non_blocking=non_blocking),
            {k: v.to(device, non_blocking=non_blocking) for k, v in self.ndata.items()},
            None if self._bne is None else self._bne.to(device, non_blocking=non_blocking),
            num_nodes=self._n,
        )
        return g

    def pin_memory(self) -> "BatchedCFG":
        g = BatchedCFG(self._src.pin_memory(), self._dst.pin_memory(), self._bnn.pin_memory(),
                       {k: v.pin_memory() for k, v in self.ndata.items()},
                       None if self._bne is None else self._bne.pin_memory(), num_nodes=self._n)
        return g

    def __repr__(self):
        return (f"BatchedCFG(batch_size={self.batch_size}, num_nodes={self._n}, "
                f"num_edges={self.num_edges()}, ndata={list(self.ndata)}, device={self.device})")


def graph(edges, num_nodes: Optional[int] = None, ndata=None) -> BatchedCFG:
    """``dgl.graph((src, dst))`` for one graph (reference ``dbize_graphs.py:24``)."""
    src, dst = edges
    src = torch.as_tensor(src, dtype=torch.int64)
    dst = torch.as_tensor(dst, dtype=torch.int64)
    if num_nodes is None:
        num_nodes = int(max(src.max().item(), dst.max().item())) + 1 if src.numel() else 0
    return BatchedCFG(src, dst, torch.tensor([num_nodes], dtype=torch.int64), ndata,
                      torch.tensor([src.numel()], dtype=torch.int64))


def add_self_loop(g: BatchedCFG) -> BatchedCFG:
    """``dgl.add_self_loop`` (reference ``dbize_graphs.py:25``): appends one ``v -> v`` edge per node."""
    n = g.num_nodes()
    loops = torch.arange(n, dtype=g._src.dtype, device=g.device)
    bne = None
    if g._bne is not None:
        bne = g._bne + g._bnn
    return BatchedCFG(torch.cat([g._src, loops]), torch.cat([g._dst, loops]), g._bnn, g.ndata, bne)


def batch(graphs: Sequence[BatchedCFG]) -> BatchedCFG:
    """``dgl.batch``: concatenate graphs, offsetting node ids (reference ``dataset.py:76``)."""
    if len(graphs) == 0:
        raise ValueError("cannot batch an empty list of graphs")
    srcs, dsts, bnns, bnes = [], [], [], []
    off = 0
    for g in graphs:
        srcs.append(g._src + off)
        dsts.append(g._dst + off)
        bnns.append(g._bnn)
        bnes.append(g.batch_num_edges())
        off += g.num_nodes()
    keys = list(graphs[0].ndata)
    ndata = {k: torch.cat([g.ndata[k] for g in graphs]) for k in keys}
    return BatchedCFG(torch.cat(srcs), torch.cat(dsts), torch.cat(bnns), ndata, torch.cat(bnes))


def unbatch(g: BatchedCFG, node_split=None) -> List[BatchedCFG]:
    """``dgl.unbatch`` (reference ``base_module.py:87``). Kept for compatibility; the CUDA path
    never unbatches (labels are a fused segment-max)."""
    bnn_t = g.batch_num_nodes().cpu().to(torch.int64)
    bnn = bnn_t.tolist()
    B = len(bnn)
    # edges of a batched graph are grouped per graph only if it came from batch(); handle the general case: an edge belongs to
    # the graph that owns its dst (dst past the last node: to none), and one stable sort keeps each graph's edges in their order
    src, dst = g.edges()
    ptr = torch.zeros(B + 1, dtype=torch.int64)
    torch.cumsum(bnn_t, 0, out=ptr[1:])
    gid = torch.bucketize(dst.cpu().to(torch.int64), ptr[1:], right=True)
    bne_t = torch.bincount(gid, minlength=B + 1)[:B]
    owned = int(bne_t.sum())
    order = torch.sort(gid, stable=True).indices[:owned].to(src.device)
    shift = torch.repeat_interleave(ptr[:-1], bne_t).to(device=src.device, dtype=src.dtype)   # first node of each edge's graph
    src, dst = src[order] - shift, dst[order] - shift.to(dst.dtype)
    eptr = [0] + bne_t.cumsum(0).tolist()
    n0 = 0
    out = []
    for b, nn_ in enumerate(bnn):
        e0, e1 = eptr[b], eptr[b + 1]
        nd = {k: v[n0:n0 + nn_] for k, v in g.ndata.items()}
        out.append(BatchedCFG(src[e0:e1], dst[e0:e1], bnn_t[b:b + 1], nd, bne_t[b:b + 1], num_nodes=nn_))
        n0 += nn_
    return out


def as_batched_cfg(g) -> BatchedCFG:
    """Adapter for a real ``dgl.DGLGraph`` (SURVEY.md §8b 'Graph argument')."""
    if isinstance(g, BatchedCFG):
        return g
    if all(hasattr(g, a) for a in ("edges", "batch_num_nodes", "ndata")):
        # memoised on the source object: a step calls this 2-3 times (forward, loss/labels) and the wrapper carries the device
        # CSR cache — a fresh wrapper per call would rebuild the CSR each time
        cached = getattr(g, "_ddfa_b200_cfg", None)
        nd = {k: g.ndata[k] for k in g.ndata.keys()}
        if cached is not None and cached.ndata.keys() == nd.keys() and \
                all(cached.ndata[k].data_ptr() == v.data_ptr() and cached.ndata[k].shape == v.shape for k, v in nd.items()):
            return cached      # same node data storage: the graph object was not re-populated since
        src, dst = g.edges()
        out = BatchedCFG(src, dst, g.batch_num_nodes(), nd)
        try:
            g._ddfa_b200_cfg = out
        except Exception:      # objects that refuse new attributes: no memoisation
            pass
        return out
    raise TypeError(f"expected a BatchedCFG or DGLGraph-like object, got {type(g)!r}")


def collate(samples: Iterable):
    """Collate ``(graph, extrafeats)`` tuples as DGL's ``GraphDataLoader`` does
    (reference ``datamodule.py:116-141``; consumer ``base_module.py:172``)."""
    graphs, extras = zip(*samples)
    merged = {}
    for k in extras[0] if extras and extras[0] else {}:
        merged[k] = torch.stack([torch.as_tensor(e[k]) for e in extras])
    return batch(list(graphs)), merged


def partition_graphs(batch_num_nodes: torch.Tensor, world_size: int):
    """Contiguous, node-count-balanced split of a batch's graphs over ``world_size`` ranks
    (SURVEY.md §8e).  Returns ``world_size + 1`` graph offsets; rank r owns graphs [off[r], off[r+1]).
    Every rank receives at least one graph when B >= world_size."""
    bnn = batch_num_nodes.to(torch.int64).cpu()
    B = int(bnn.shape[0])
    if world_size < 1:
        raise ValueError("world_size must be >= 1")
    if B < world_size:
        raise ValueError(f"cannot split {B} graphs over {world_size} ranks")
    csum = torch.cumsum(bnn, 0)
    total = int(csum[-1]) if B else 0
    offs = [0]
    for r in range(1, world_size):
        target = total * r / world_size
        cut = int(torch.searchsorted(csum, torch.tensor(target, dtype=csum.dtype), right=False)) + 1
        cut = max(cut, offs[-1] + 1)              # at least one graph per rank
        cut = min(cut, B - (world_size - r))      # leave one graph for each remaining rank
        offs.append(cut)
    offs.append(B)
    return offs


def slice_batch(g: BatchedCFG, g0: int, g1: int) -> BatchedCFG:
    """Graphs [g0, g1) of a batch as a new batch (node ids re-based).  Pure tensor slicing on the
    graph's device: node ids of a batch are contiguous per graph."""
    bnn = g.batch_num_nodes()
    ptr = torch.zeros(bnn.shape[0] + 1, dtype=torch.int64, device=bnn.device)
    ptr[1:] = torch.cumsum(bnn, 0)
    n0, n1 = int(ptr[g0]), int(ptr[g1])
    src, dst = g.edges()
    keep = ((dst >= n0) & (dst < n1)).nonzero().squeeze(-1)
    nd = {k: v[n0:n1] for k, v in g.ndata.items()}
    return BatchedCFG(src[keep] - n0, dst[keep] - n0, bnn[g0:g1].clone(), nd)


def split_batch(g: BatchedCFG, world_size: int) -> List[BatchedCFG]:
    """Shard a batch over ranks (no data-path collective is needed: graphs never exchange messages)."""
    offs = partition_graphs(g.batch_num_nodes(), world_size)
    return [slice_batch(g, offs[r], offs[r + 1]) for r in range(world_size)]
