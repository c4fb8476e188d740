"""Restatement of the CSV rules ``bigvul_io.load_arena`` parses on the device (``csrc/csv_load.cu``), and of the arena it lays
out (not a test module).  Shared by tests/test_csv_rule_cpu.py, which holds the CSV rules to ``pandas.read_csv``, and
tests/test_csv_load_gpu.py, which holds the device loader to both.

- ``row_spans``: a row ends at a ``\\n`` with an even number of ``"`` before it (a ``""`` escape toggles twice); a final row
  without its newline counts; blank lines are skipped; the bytes of a row are those after the previous row's end, blank lines
  dropped, without the ``\\r`` of a ``\\r\\n``.
- ``split_fields``: commas outside quotes separate the fields of a row.
- ``to_int``: a field that is a signed decimal integer, optionally quoted, optionally followed by ``.`` and zeros (an integral
  float), in int64; anything else is ``None``.
- ``read_columns``: the named columns of every data row as int64 arrays (the header is the first row).
- ``arena_rule``: from the parsed columns, what ``GraphArena.from_graphs([load_graphs(...)[i] for i in sorted ids])`` holds,
  with NumPy (the graphs in ascending graph_id, nodes and edges in file row order, self-loops appended, features left-joined
  on (graph_id, node_id), ``_VULN`` through fp32).
"""
import re

import numpy as np

_INT = re.compile(rb"[+-]?[0-9]+(\.0*)?")


def row_spans(data: bytes):
    """[(start, end)] byte ranges of the non-blank rows, header included."""
    if not data.endswith(b"\n"):
        data += b"\n"
    b = np.frombuffer(data, np.uint8)
    n = b.shape[0]
    quote = b == ord('"')
    before = np.cumsum(quote) - quote                      # quotes before each byte
    nl = np.flatnonzero((b == 10) & (before % 2 == 0))
    prev1 = np.where(nl >= 1, b[np.maximum(nl - 1, 0)], 10)
    prev2 = np.where(nl >= 2, b[np.maximum(nl - 2, 0)], 10)
    blank = (nl == 0) | (prev1 == 10) | ((prev1 == 13) & (prev2 == 10))
    ends = nl[~blank]
    starts = np.concatenate([[0], ends[:-1] + 1]).astype(np.int64)
    eol = (b == 10) | (b == 13)
    nxt = np.minimum.accumulate(np.where(eol, n, np.arange(n))[::-1])[::-1]       # next byte that is not \r or \n
    starts = np.minimum(nxt[np.minimum(starts, n - 1)], ends)
    ends = ends - ((ends > starts) & (b[np.maximum(ends - 1, 0)] == 13))
    return [(int(s), int(e)) for s, e in zip(starts, ends)], data


def split_fields(row: bytes):
    out, start, inq = [], 0, False
    for i, ch in enumerate(row):
        if ch == 34:
            inq = not inq
        elif ch == 44 and not inq:
            out.append(row[start:i])
            start = i + 1
    out.append(row[start:])
    return out


def unquote(field: bytes) -> str:
    if len(field) >= 2 and field[:1] == b'"' and field[-1:] == b'"':
        field = field[1:-1].replace(b'""', b'"')
    return field.decode("utf-8")


def to_int(field: bytes):
    if len(field) >= 2 and field[:1] == b'"' and field[-1:] == b'"':
        field = field[1:-1]
    if not _INT.fullmatch(field):
        return None
    v = int(field.split(b".")[0])
    return v if -2 ** 63 <= v < 2 ** 63 else None


def read_columns(data: bytes, names):
    """{name: int64 array} over the data rows; raises ValueError(line, name) at the first bad field."""
    spans, data = row_spans(data)
    header = [unquote(f) for f in split_fields(data[spans[0][0]:spans[0][1]])]
    pos = {name: header.index(name) for name in names}
    out = {name: np.empty(len(spans) - 1, np.int64) for name in names}
    for r, (s, e) in enumerate(spans[1:]):
        fields = split_fields(data[s:e])
        for name in names:
            v = to_int(fields[pos[name]]) if pos[name] < len(fields) else None
            if v is None:
                raise ValueError(data[:s].count(b"\n") + 1, name)
            out[name][r] = v
    return out


def arena_rule(nodes, edges, features):
    """nodes: {graph_id, node_id, vuln}, edges: {graph_id, innode, outnode}, features: [(ndata key, {graph_id, node_id, value})]
    -> dict of NumPy arrays (graph_ids, nodes_per_graph, edges_per_graph, node_off, src, dst, feats, vuln, CSR)."""
    order = np.argsort(nodes["graph_id"], kind="stable")
    gsorted = nodes["graph_id"][order]
    gids, first, npg = np.unique(gsorted, return_index=True, return_counts=True)
    eorder = np.argsort(edges["graph_id"], kind="stable")
    esorted = edges["graph_id"][eorder]
    lo, hi = np.searchsorted(esorted, gids, "left"), np.searchsorted(esorted, gids, "right")
    ne = hi - lo
    node_off = np.concatenate([[0], np.cumsum(npg)])
    sel = np.concatenate([eorder[a:b] for a, b in zip(lo, hi)]) if len(gids) else np.zeros(0, np.int64)
    shift = np.repeat(node_off[:-1], ne)
    e_src, e_dst = edges["innode"][sel] + shift, edges["outnode"][sel] + shift
    # per graph: its edge rows then its self-loops
    epg = ne + npg
    eoff = np.concatenate([[0], np.cumsum(epg)])
    E = int(eoff[-1])
    src, dst = np.empty(E, np.int64), np.empty(E, np.int64)
    is_edge = np.zeros(E, bool)
    is_edge[np.repeat(eoff[:-1], ne) + (np.arange(ne.sum()) - np.repeat(np.cumsum(ne) - ne, ne))] = True
    src[is_edge], dst[is_edge] = e_src, e_dst
    loops = np.arange(int(node_off[-1]))
    src[~is_edge], dst[~is_edge] = loops, loops
    feats = {}
    for key, f in features:
        # (graph_id, node_id) as one int64 key (the test data keeps both ranges small enough)
        g0 = min(f["graph_id"].min(), nodes["graph_id"].min())
        k0 = min(f["node_id"].min(), nodes["node_id"].min())
        span = int(max(f["node_id"].max(), nodes["node_id"].max()) - k0 + 1)
        assert (int(max(f["graph_id"].max(), nodes["graph_id"].max()) - g0) + 1) * span < 2 ** 62
        fkey = (f["graph_id"] - g0) * span + (f["node_id"] - k0)
        nkey = (nodes["graph_id"][order] - g0) * span + (nodes["node_id"][order] - k0)
        fo = np.argsort(fkey, kind="stable")
        pos = np.searchsorted(fkey[fo], nkey)
        assert (fkey[fo][np.minimum(pos, len(fo) - 1)] == nkey).all(), "a node without a feature row"
        feats[key] = f["value"][fo][pos]
    vuln = nodes["vuln"][order].astype(np.float32).astype(np.int32)
    N = int(node_off[-1])
    o = np.lexsort((src, dst))
    indptr = np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=N))]).astype(np.int32)
    ot = np.lexsort((dst, src))
    indptr_t = np.concatenate([[0], np.cumsum(np.bincount(src, minlength=N))]).astype(np.int32)
    return dict(graph_ids=gids, nodes_per_graph=npg.astype(np.int64), edges_per_graph=epg.astype(np.int64),
                node_off=node_off.astype(np.int32), src=src, dst=dst, feats=feats, vuln=vuln,
                indptr=indptr, indices=src[o].astype(np.int32), indptr_t=indptr_t, indices_t=dst[ot].astype(np.int32))
