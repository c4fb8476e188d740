"""DGL-free reader of the reference's processed Big-Vul files (SURVEY.md §8 row f2) -> graphs -> :class:`GraphArena`.

What the reference does, and where:

* ``DDFA/sastvd/scripts/dbize.py:40-60,104-105`` writes ``nodes.csv`` (one row per CFG node: ``graph_id, node_id, dgl_id, vuln,
  code, _label``; ``dgl_id`` = row number inside the graph) and ``edges.csv`` (``graph_id, innode, outnode`` in dgl ids).
* ``DDFA/sastvd/scripts/dbize_graphs.py:17-33`` turns every graph's edge rows into ``dgl.graph((innode, outnode))`` — so the
  message source is ``innode`` and the destination ``outnode``, and the node count is ``max id + 1`` — then
  ``dgl.add_self_loop`` (one ``v -> v`` edge per node, appended), and saves ``graphs.bin``.
* ``DDFA/sastvd/scripts/dbize_absdf.py`` writes ``nodes_feat_<feat>_fixed.csv`` (``graph_id, node_id, <feat>``): the
  abstract-dataflow vocabulary index of every node (0 = not a definition, 1 = unknown, 2.. = known).
* ``DDFA/sastvd/linevd/graphmogrifier.py:20-40`` left-merges the feature file(s) onto ``nodes.csv`` by ``(graph_id, node_id)``
  (``concat_all_absdf``: the four ``_ABS_DATAFLOW_{api,datatype,literal,operator}...`` files, renamed to
  ``_ABS_DATAFLOW_<subkey>``); ``:59-95`` attaches, per graph in ``groupby("graph_id")`` order and in FILE ROW ORDER inside
  the graph, ``ndata["_ABS_DATAFLOW"]``, the four subkey vectors and ``ndata["_VULN"]``; graphs without node rows are dropped.
* ``DDFA/sastvd/helpers/dclass.py:84-105`` draws the per-epoch index set (``undersample="v1.0"``: all vulnerable examples plus
  as many non-vulnerable ones, sampled without replacement from a persistent ``RandomState``).

This module restates exactly that with pandas (the ``.bin`` container itself is DGL's and is not read: it holds nothing that
``edges.csv`` does not).  The dataset is not shipped with the reference, so the tests build small files in the same schema —
and the reference's OWN ``get_nodes_df`` / ``get_graphs`` / ``get_epoch_indices`` were run on those files in the build container
(``tests/golden/make_reference_io_golden.py``); ``tests/test_bigvul_io.py::test_reader_matches_reference_loaders`` holds the
reader to their output.  Only the three DGL calls of ``dbize_graphs.py`` stay a restatement.
"""
from __future__ import annotations

import csv
import ctypes as C
import io
from pathlib import Path
from typing import Dict, Optional, Tuple

import numpy as np
import pandas as pd
import torch

from . import _lib
from . import engine as E
from .batched_graph import ABS_DATAFLOW_SUBKEYS, BatchedCFG, add_self_loop, graph


def _sample_text(sample_mode: bool) -> str:
    return "_sample" if sample_mode else ""


def read_edge_graphs(edges_csv) -> Dict[int, BatchedCFG]:
    """``dbize_graphs.py:17-27``: one graph per ``graph_id`` (in ``groupby`` = ascending id order), self-loops appended."""
    df = pd.read_csv(edges_csv, index_col=0, usecols=["Unnamed: 0", "graph_id", "innode", "outnode"])
    out: Dict[int, BatchedCFG] = {}
    for graph_id, group in df.groupby("graph_id"):
        g = graph((group["innode"].tolist(), group["outnode"].tolist()))     # src = innode, dst = outnode, N = max id + 1
        out[int(graph_id)] = add_self_loop(g)
    return out


def read_nodes(processed_dir, dsname: str = "bigvul", feat: Optional[str] = None, concat_all_absdf: bool = False,
               sample_mode: bool = False, load_features: bool = True) -> pd.DataFrame:
    """Node table with the requested feature columns merged in — the semantics of ``graphmogrifier.get_nodes_df`` (:20-40):
    every feature file is LEFT-joined on ``(graph_id, node_id)``, so node order is that of ``nodes.csv``."""
    folder = Path(processed_dir) / dsname
    tag = _sample_text(sample_mode)
    table = pd.read_csv(folder / f"nodes{tag}.csv", index_col=0, dtype={"code": str}, na_values=[],
                        usecols=["Unnamed: 0", "graph_id", "node_id", "dgl_id", "vuln", "code", "_label"]).reset_index(drop=True)
    table["code"] = table["code"].astype(str)
    if not load_features:
        return table
    joins = []                                           # (file stem, column rename or None)
    if feat is not None:
        joins.append((feat, None))
    if concat_all_absdf:
        tail = feat[feat.index("_all"):]                 # e.g. "_all_limitall_1000_limitsubkeys_1000"
        joins += [(f"_ABS_DATAFLOW_{sub}{tail}", f"_ABS_DATAFLOW_{sub}") for sub in ABS_DATAFLOW_SUBKEYS]
    for stem, new_name in joins:
        extra = pd.read_csv(folder / f"nodes_feat_{stem}_fixed{tag}.csv", index_col=0)
        if new_name is not None:
            first = [c for c in extra.columns if c.startswith("_ABS_DATAFLOW")][0]
            extra = extra.rename(columns={first: new_name})
        table = table.merge(extra, how="left", on=["graph_id", "node_id"])
    return table


def attach_node_data(graphs_by_id: Dict[int, BatchedCFG], nodes: pd.DataFrame, feat: str, concat_all_absdf: bool = False
                     ) -> Dict[int, BatchedCFG]:
    """``graphmogrifier.get_graphs`` (:59-95): ndata per graph in file row order; graphs without node rows are dropped."""
    out: Dict[int, BatchedCFG] = {}
    for graph_id, group in nodes.groupby("graph_id"):
        g = graphs_by_id[int(graph_id)]
        if len(group) != g.num_nodes():
            # DGL raises here too (ndata length must equal the node count)
            raise ValueError(f"graph {graph_id}: {len(group)} node rows but the edge list implies {g.num_nodes()} nodes")
        ndata = {"_ABS_DATAFLOW": torch.LongTensor(group[feat].tolist())}
        if concat_all_absdf:
            for other in ABS_DATAFLOW_SUBKEYS:
                ndata[f"_ABS_DATAFLOW_{other}"] = torch.LongTensor(group[f"_ABS_DATAFLOW_{other}"].tolist())
        ndata["_VULN"] = torch.Tensor(group["vuln"].tolist()).int()
        src, dst = g.edges()
        out[int(graph_id)] = BatchedCFG(src, dst, g.batch_num_nodes(), ndata, g.batch_num_edges(), num_nodes=g.num_nodes())
    return out


def load_graphs(processed_dir, dsname: str = "bigvul", feat: Optional[str] = None, concat_all_absdf: bool = False,
                sample_mode: bool = False) -> Dict[int, BatchedCFG]:
    """edges.csv + nodes.csv + feature files -> {graph_id: single graph with ndata}, as the reference's dataset holds them."""
    base = Path(processed_dir) / dsname
    graphs = read_edge_graphs(base / f"edges{_sample_text(sample_mode)}.csv")
    nodes = read_nodes(processed_dir, dsname, feat, concat_all_absdf, sample_mode)
    return attach_node_data(graphs, nodes, feat, concat_all_absdf)


def load_arena(processed_dir, device="cuda", dsname: str = "bigvul", feat: Optional[str] = None, concat_all_absdf: bool = False,
               sample_mode: bool = False) -> Tuple["object", np.ndarray]:
    """The whole processed dataset as a device-resident :class:`deepdfa_b200.GraphArena`, built on the device from the files'
    bytes (``csrc/csv_load.cu``); returns (arena, graph_ids) with ``graph_ids[i]`` = the reference's id of arena graph ``i``
    (ascending).  The arena is bit-identical to ``GraphArena.from_graphs([load_graphs(...)[i] for i in sorted ids])``.

    Inconsistent or malformed files raise ``ValueError`` naming the file and the line or graph: a token that is not an
    integer, a missing column, an unterminated quote, a node-row graph without edge rows, a negative endpoint, a node count
    other than the edge list's ``max id + 1``, a node without a feature row or with two, more than 2^31 nodes or edges, a
    file larger than the free device memory.  No device memory stays allocated after an error."""
    message = None
    try:
        return _DeviceLoad(processed_dir, device, dsname, feat, concat_all_absdf, sample_mode).run()
    except _LoadError as e:
        message = str(e)      # raised below, outside this frame's handler: the traceback then holds no device tensor
    raise ValueError(message)


class _LoadError(Exception):
    pass


_ROW_LIMIT = 2 ** 31


def _header(host: np.ndarray) -> list:
    """The first non-blank row of a CSV file's bytes, as names."""
    text = bytes(host[: 1 << 20]).decode("utf-8", "replace")
    for row in csv.reader(io.StringIO(text, newline="")):
        if row:
            return row
    return []


class _DeviceLoad:
    """One ``load_arena`` call: every file read into pinned memory, copied to the device, indexed and parsed there, its bytes
    freed before the next file; then the graphs grouped, the union COO laid out and the feature files joined on the device.
    Host syncs: two per file (row count; parse errors and column ranges), one after grouping, one per feature file after its
    join, one for the arena's host copies of the graph sizes — none per graph."""

    def __init__(self, processed_dir, device, dsname, feat, concat_all_absdf, sample_mode):
        if feat is None:
            raise _LoadError("load_arena: feat (the feature file whose column becomes _ABS_DATAFLOW) is required")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _LoadError(f"load_arena: device must be CUDA, got {dev}")
        self.dev = dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())
        self.folder = Path(processed_dir) / dsname
        self.tag = _sample_text(sample_mode)
        # (ndata key, file, column name, whether the name is a prefix): attach_node_data's key order
        self.features = [("_ABS_DATAFLOW", self.folder / f"nodes_feat_{feat}_fixed{self.tag}.csv", feat, False)]
        if concat_all_absdf:
            tail = feat[feat.index("_all"):]
            self.features += [(f"_ABS_DATAFLOW_{sub}", self.folder / f"nodes_feat__ABS_DATAFLOW_{sub}{tail}_fixed{self.tag}.csv",
                               "_ABS_DATAFLOW", True) for sub in ABS_DATAFLOW_SUBKEYS]
        self.L = _lib.lib()

    # ------------------------------------------------------------------------------------------------
    def _empty(self, n, dtype):
        return torch.empty(int(n), dtype=dtype, device=self.dev)

    def _parse(self, path: Path, columns):
        """columns: [(name, is_prefix)] -> (data rows, [int64 tensor per column], [(min, max) per column])."""
        from ._lib import ptr_array
        L, st = self.L, E._stream_ptr()
        if not path.exists():
            raise _LoadError(f"{path}: no such file")
        size = path.stat().st_size
        host = torch.empty(size + 1, dtype=torch.uint8, pin_memory=True)
        hnp = host.numpy()
        with open(path, "rb") as f:
            got = f.readinto(memoryview(hnp[:size]))
        if got != size:
            raise _LoadError(f"{path}: read {got} of {size} bytes")
        n = size
        if n == 0 or hnp[n - 1] != 10:           # a final row without its newline
            hnp[n] = 10
            n += 1
        names = _header(hnp[:n])
        positions = []
        for name, is_prefix in columns:
            # a prefix: read_nodes' "first column starting with _ABS_DATAFLOW" among the columns after the index column
            found = [i for i, c in enumerate(names) if (c.startswith(name) and i > 0 if is_prefix else c == name)]
            if not found:
                raise _LoadError(f"{path}: no column {'starting with ' if is_prefix else ''}{name!r} in the header {names}")
            positions.append(found[0])
        padded = (n + 15) // 16 * 16
        ws_bytes = L.call("ddfa_csv_index_workspace_bytes", n)
        free = torch.cuda.mem_get_info(self.dev)[0] + torch.cuda.memory_reserved(self.dev) - torch.cuda.memory_allocated(self.dev)
        if padded + ws_bytes > free:
            raise _LoadError(f"{path}: {size} bytes do not fit in the {free} bytes of free device memory (files are not streamed)")
        text = self._empty(padded, torch.uint8)
        text[:n].copy_(host[:n], non_blocking=True)
        ws = self._empty(ws_bytes, torch.uint8)
        info = self._empty(2, torch.int64)
        L.call("ddfa_csv_index_count", text.data_ptr(), n, info.data_ptr(), ws.data_ptr(), ws_bytes, st)
        rows, parity = info.tolist()
        row_end = self._empty(max(rows, 1), torch.int64)
        if rows:
            L.call("ddfa_csv_index_rows", text.data_ptr(), n, row_end.data_ptr(), ws.data_ptr(), ws_bytes, st)
        del ws

        def line_of(byte):                       # 1-based line of the first non-blank byte at or after `byte`
            while byte < n and hnp[byte] in (10, 13):
                byte += 1
            return int(np.count_nonzero(hnp[:byte] == 10)) + 1

        if parity:
            start = int(row_end[rows - 1]) + 1 if rows else 0
            raise _LoadError(f"{path}, line {line_of(start)}: unterminated quote")
        if rows == 0:
            raise _LoadError(f"{path}: no header row")
        data = rows - 1
        if data >= _ROW_LIMIT:
            raise _LoadError(f"{path}: {data} rows, more than 2^31 nodes or edges")
        uniq = sorted(set(positions))
        outs = {pos: self._empty(max(data, 1), torch.int64) for pos in uniq}
        finfo = self._empty(1 + 2 * len(uniq), torch.int64)
        L.call("ddfa_csv_fields", text.data_ptr(), row_end.data_ptr(), rows, (C.c_int32 * len(uniq))(*uniq), len(uniq),
               ptr_array([outs[pos].data_ptr() for pos in uniq]), finfo.data_ptr(), st)
        fi = finfo.tolist()
        bad = fi[0] & (2 ** 64 - 1)
        if bad != 2 ** 64 - 1:
            r, reason, slot = bad >> 8, (bad >> 4) & 15, bad & 15
            what = "not an integer" if reason == _lib.CSV_ERR_NOT_INT else "the row has no such field"
            line = line_of(int(row_end[r]) + 1)
            raise _LoadError(f"{path}, line {line}, column {names[uniq[slot]]!r}: {what}")
        del text, row_end, host
        ranges = {pos: (fi[1 + 2 * k], fi[2 + 2 * k]) for k, pos in enumerate(uniq)}
        return data, [outs[p][:data] for p in positions], [ranges[p] for p in positions]

    def _sort(self, n, major, major_range, minor=None, minor_range=(0, 0)):
        """Row ids 0 .. n-1 stably sorted by (major, minor)."""
        L = self.L
        perm = self._empty(max(n, 1), torch.int32)
        if n == 0:
            return perm
        ws = self._empty(L.call("ddfa_row_sort_workspace_bytes", n), torch.uint8)
        bits = lambda r: max(r[1] - r[0], 0).bit_length()
        L.call("ddfa_row_sort", major.data_ptr(), major_range[0], bits(major_range), 0 if minor is None else minor.data_ptr(),
               minor_range[0], 0 if minor is None else bits(minor_range), n, perm.data_ptr(), ws.data_ptr(), ws.numel(), E._stream_ptr())
        return perm

    # ------------------------------------------------------------------------------------------------
    def run(self):
        from ._lib import ptr_array
        from .arena import GraphArena
        L = self.L
        with torch.cuda.device(self.dev):
            st = E._stream_ptr()
            nodes_csv = self.folder / f"nodes{self.tag}.csv"
            edges_csv = self.folder / f"edges{self.tag}.csv"
            rn, (ngid, nnid, nvul), (ngid_r, _, _) = self._parse(nodes_csv, [("graph_id", False), ("node_id", False), ("vuln", False)])
            if rn == 0:
                raise _LoadError(f"{nodes_csv}: no node rows")
            node_perm = self._sort(rn, ngid, ngid_r)
            re_, (egid, ein, eout), (egid_r, _, _) = self._parse(edges_csv, [("graph_id", False), ("innode", False), ("outnode", False)])
            edge_perm = self._sort(re_, egid, egid_r)

            gws = self._empty(L.call("ddfa_csv_graphs_workspace_bytes", rn), torch.uint8)
            ginfo = self._empty(_lib.CSV_GRAPH_INFO_WORDS, torch.int64)
            L.call("ddfa_csv_graphs", ngid.data_ptr(), node_perm.data_ptr(), rn, egid.data_ptr(), edge_perm.data_ptr(), re_,
                   ein.data_ptr(), eout.data_ptr(), ginfo.data_ptr(), gws.data_ptr(), gws.numel(), st)
            gi = ginfo.tolist()
            bad = gi[2] & (2 ** 64 - 1)
            if bad != 2 ** 64 - 1:
                reason, implied, rows, gid = (bad >> 4) & 15, gi[3], gi[4], gi[5]
                if reason == _lib.CSV_ERR_NO_EDGES:
                    raise _LoadError(f"{edges_csv}: graph {gid} has {rows} node rows in {nodes_csv.name} but no edge rows")
                if reason == _lib.CSV_ERR_NEGATIVE:
                    raise _LoadError(f"{edges_csv}: graph {gid} has a negative endpoint")
                raise _LoadError(f"{nodes_csv}: graph {gid}: {rows} node rows but the edge list of {edges_csv.name} implies {implied} nodes")
            G, Eu = gi[0], gi[1]
            if Eu >= _ROW_LIMIT:
                raise _LoadError(f"{edges_csv}: {Eu} edges with the self-loops, more than 2^31 nodes or edges")
            src, dst = self._empty(max(Eu, 1), torch.int32), self._empty(max(Eu, 1), torch.int32)
            vuln = self._empty(rn, torch.int32)
            npg, epg, gids = (self._empty(G, torch.int64) for _ in range(3))
            L.call("ddfa_csv_union", ngid.data_ptr(), node_perm.data_ptr(), rn, nvul.data_ptr(), edge_perm.data_ptr(), ein.data_ptr(),
                   eout.data_ptr(), G, gws.data_ptr(), gws.numel(), src.data_ptr(), dst.data_ptr(), vuln.data_ptr(), npg.data_ptr(),
                   epg.data_ptr(), gids.data_ptr(), st)
            del gws, egid, ein, eout, edge_perm, nvul

            feats = {key: self._empty(rn, torch.int64) for key, _, _, _ in self.features}
            by_file = {}
            for key, path, name, is_prefix in self.features:
                by_file.setdefault(path, []).append((key, name, is_prefix))
            for path, wanted in by_file.items():
                rf, cols, ranges = self._parse(path, [("graph_id", False), ("node_id", False)] + [(nm, pf) for _, nm, pf in wanted])
                perm = self._sort(rf, cols[0], ranges[0], cols[1], ranges[1])
                jws = self._empty(max(L.call("ddfa_csv_join_workspace_bytes", rf), 16), torch.uint8)
                jinfo = self._empty(1, torch.int64)
                L.call("ddfa_csv_join", ngid.data_ptr(), nnid.data_ptr(), node_perm.data_ptr(), rn, cols[0].data_ptr(), cols[1].data_ptr(),
                       perm.data_ptr(), rf, ptr_array([c.data_ptr() for c in cols[2:]]), len(wanted),
                       ptr_array([feats[key].data_ptr() for key, _, _ in wanted]), jinfo.data_ptr(), jws.data_ptr(), jws.numel(), st)
                bad = int(jinfo.item()) & (2 ** 64 - 1)
                if bad != 2 ** 64 - 1:
                    i, reason = bad >> 8, (bad >> 4) & 15
                    r = int(node_perm[i])
                    what = "no feature row" if reason == _lib.CSV_ERR_NO_FEATURE else "more than one feature row"
                    raise _LoadError(f"{path}: {what} for graph {int(ngid[r])}, node {int(nnid[r])}")
                del cols, perm, jws
            del ngid, nnid, node_perm

            ndata = dict(feats)
            ndata["_VULN"] = vuln
            big = BatchedCFG(src[:Eu], dst[:Eu], npg, ndata, epg, num_nodes=rn)
            arena = GraphArena.from_union(big, self.dev)
            return arena, gids.cpu().numpy()


def epoch_indices(df: pd.DataFrame, undersample=None, oversample=None, rng: Optional[np.random.RandomState] = None) -> pd.Index:
    """Index set of one epoch — ``BigVulDataset.get_epoch_indices`` (dclass.py:84-105).  ``df``: one row per example with a
    0/1 column ``vul``; ``rng``: the dataset's persistent ``np.random.RandomState(seed)`` (successive epochs draw different
    subsets).  ``undersample="v<f>"`` keeps ``int(f * #vulnerable)`` non-vulnerable rows, a float keeps that fraction of them;
    ``oversample=<f>`` redraws ``int(f * #vulnerable)`` vulnerable rows with replacement.  Draw order (non-vulnerable first,
    then vulnerable) and the result order (vulnerable rows, then non-vulnerable) follow the reference, so the same seed gives
    the same epochs."""
    if undersample is None and oversample is None:
        return df.index
    positives, negatives = df[df.vul == 1], df[df.vul == 0]
    if undersample is not None:
        spec = str(undersample)
        keep = int(len(positives) * float(spec[1:])) if spec.startswith("v") else int(len(negatives) * undersample)
        negatives = negatives.sample(keep, replace=False, random_state=rng)
    if oversample is not None:
        positives = positives.sample(int(len(positives) * oversample), replace=True, random_state=rng)
    return positives.index.append(negatives.index)
