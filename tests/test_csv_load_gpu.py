"""GPU: bigvul_io.load_arena builds the arena on the device from the files' bytes (csrc/csv_load.cu).  It must be bit-identical
to the host composition GraphArena.from_graphs([load_graphs(...)[i] for i in sorted ids]) on the bigvul_fixture files, on
awkward text (quoted commas and newlines, "" escapes, \\r\\n, blank lines, permuted and extra columns, integral floats), on a
20 000-graph set, and, against the NumPy restatement of tests/csv_rule.py, at Big-Vul size; the row index and the field
parser must match the restatement with quotes and newlines on every side of the kernel's 4096-byte chunk boundaries; every
error raises ValueError and leaves no device memory allocated."""
import os
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from deepdfa_b200 import bigvul_io as IO, synth
from deepdfa_b200.arena import GraphArena

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import csv_rule as R  # noqa: E402
from bigvul_fixture import FEAT, write_dataset  # noqa: E402
from test_csv_rule_cpu import AWKWARD  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def host_arena(root, **kw):
    graphs = IO.load_graphs(root, "bigvul", **kw)
    ids = np.array(sorted(graphs), dtype=np.int64)
    return GraphArena.from_graphs([graphs[int(i)] for i in ids], DEV), ids


def assert_same(got, want):
    (a, ia), (b, ib) = got, want
    assert ia.dtype == ib.dtype and np.array_equal(ia, ib)
    assert torch.equal(a.node_off, b.node_off) and a.node_off.dtype == b.node_off.dtype
    for x, y in ((a.nodes_per_graph, b.nodes_per_graph), (a.edges_per_graph, b.edges_per_graph)):
        assert x.dtype == y.dtype and np.array_equal(x, y)
    assert list(a.feats) == list(b.feats)
    for k in a.feats:
        assert a.feats[k].dtype == b.feats[k].dtype and torch.equal(a.feats[k], b.feats[k]), k
    assert a.vuln.dtype == b.vuln.dtype and torch.equal(a.vuln, b.vuln)
    assert (a.dg.num_nodes, a.dg.num_edges, a.dg.batch_size) == (b.dg.num_nodes, b.dg.num_edges, b.dg.batch_size)
    for name in ("indptr", "indices", "indptr_t", "indices_t", "graph_ptr"):
        assert torch.equal(getattr(a.dg, name), getattr(b.dg, name)), name


def assert_rule(got, want):
    a, ids = got
    assert np.array_equal(ids, want["graph_ids"])
    assert np.array_equal(a.nodes_per_graph, want["nodes_per_graph"]) and np.array_equal(a.edges_per_graph, want["edges_per_graph"])
    assert np.array_equal(a.node_off.cpu().numpy(), want["node_off"])
    assert np.array_equal(a.vuln.cpu().numpy(), want["vuln"])
    assert list(a.feats) == list(want["feats"])
    for k, v in want["feats"].items():
        assert np.array_equal(a.feats[k].cpu().numpy(), v), k
    E = a.dg.num_edges
    for name in ("indptr", "indices", "indptr_t", "indices_t"):
        assert np.array_equal(getattr(a.dg, name).cpu().numpy()[: E if "indices" in name else None], want[name]), name


def add_sample_tag(root):
    for p in (root / "bigvul").iterdir():
        p.rename(p.with_name(p.stem + "_sample.csv"))


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("concat", [False, True])
@pytest.mark.parametrize("sample_mode", [False, True])
def test_fixture_matches_host_composition(tmp_path, seed, concat, sample_mode):
    write_dataset(tmp_path, seed=seed, n_graphs=7 + 40 * seed)
    if sample_mode:
        add_sample_tag(tmp_path)
    kw = dict(feat=FEAT, concat_all_absdf=concat, sample_mode=sample_mode)
    assert_same(IO.load_arena(tmp_path, DEV, **kw), host_arena(tmp_path, **kw))


def rewrite_awkward(root, seed):
    """The fixture's files rewritten with awkward text: code strings with quotes, commas, newlines and multibyte UTF-8,
    \\r\\n line ends, blank lines, permuted and extra columns, integral floats, no final newline."""
    rng = np.random.default_rng(seed)
    folder = root / "bigvul"
    nodes = pd.read_csv(folder / "nodes.csv", index_col=0)
    nodes["code"] = [AWKWARD[i] + "x" * int(rng.integers(0, 40)) for i in rng.integers(0, len(AWKWARD), len(nodes))]
    nodes["lineNumber"] = rng.random(len(nodes))
    cols = list(nodes.columns)
    rng.shuffle(cols)
    text = nodes[cols].to_csv(lineterminator="\r\n")
    lines = text.split("\r\n")
    for i in sorted(rng.choice(len(lines), 5, replace=False), reverse=True):
        lines.insert(int(i) + 1, "")                   # blank lines (never inside a quoted field: those hold a \r\n too)
    (folder / "nodes.csv").write_bytes("\r\n".join(lines).encode("utf-8"))
    edges = (folder / "edges.csv").read_bytes()
    (folder / "edges.csv").write_bytes(b"\n" + edges.rstrip(b"\n"))
    for p in folder.glob("nodes_feat_*"):
        df = pd.read_csv(p, index_col=0)
        col = [c for c in df.columns if c.startswith("_ABS")][0]
        df[col] = df[col].astype(float)                # "5.0"
        df[f"note{col}"] = "x,y"                       # an extra column per file (one name in several files breaks the host merges)
        df.to_csv(p)


@pytest.mark.parametrize("seed", [0, 1])
def test_awkward_text_matches_host_composition(tmp_path, seed):
    write_dataset(tmp_path, seed=seed, n_graphs=400)
    rewrite_awkward(tmp_path, seed)
    kw = dict(feat=FEAT, concat_all_absdf=True)
    assert_same(IO.load_arena(tmp_path, DEV, **kw), host_arena(tmp_path, **kw))


@pytest.mark.parametrize("where", ["quote", "escape", "newline", "crlf", "comma"])
def test_row_index_across_chunk_boundaries(tmp_path, where):
    """A quoted code field holding the awkward bytes, moved byte by byte across the 4096-byte chunk and 16-byte thread edges."""
    payload = {"quote": '"', "escape": '""', "newline": "\n", "crlf": "\r\n", "comma": ","}[where]
    loader = IO._DeviceLoad(tmp_path, DEV, "bigvul", FEAT, False, False)
    header = ",graph_id,code,node_id\n"
    for pad in range(4096 - 40, 4096 + 24):
        rows = [header]
        filler = "y" * (pad - len(header) - len("0,1,,2\n"))
        rows.append(f"0,1,{filler},2\n")
        code = '"' + ("a" + payload.replace('"', '""') + "b") * 3 + '"'
        for r in range(1, 40):
            rows.append(f"{r},{r + 1},{code},{-r}\n" if r % 3 else f"\n{r},{r + 1},{code},{-r}\r\n")
        data = "".join(rows).encode()
        p = tmp_path / f"t{pad}.csv"
        p.write_bytes(data)
        want = R.read_columns(data, ["graph_id", "node_id"])
        n, cols, _ = loader._parse(p, [("graph_id", False), ("node_id", False)])
        assert n == len(want["graph_id"]), pad
        assert cols[0].cpu().numpy().tolist() == want["graph_id"].tolist(), pad
        assert cols[1].cpu().numpy().tolist() == want["node_id"].tolist(), pad


def test_20k_graphs_match_host_composition(tmp_path):
    synth.write_bigvul_files(tmp_path, 20_000, seed=5, mu=3.3, sigma=0.7, big_graph=800)
    feat = f"_ABS_DATAFLOW_datatype{synth.BIGVUL_TAIL}"
    kw = dict(feat=feat, concat_all_absdf=True)
    assert_same(IO.load_arena(tmp_path, DEV, **kw), host_arena(tmp_path, **kw))


def test_bigvul_size_matches_restatement(tmp_path):
    t = synth.write_bigvul_files(tmp_path, 190_000, seed=11)
    assert t["nodes"]["graph_id"].shape[0] >= 10_000_000
    feat = f"_ABS_DATAFLOW_api{synth.BIGVUL_TAIL}"
    got = IO.load_arena(tmp_path, DEV, feat=feat, concat_all_absdf=True)
    feats = [("_ABS_DATAFLOW", t["features"]["api"])] + [(f"_ABS_DATAFLOW_{s}", t["features"][s]) for s in ("api", "datatype", "literal", "operator")]
    want = R.arena_rule(t["nodes"], t["edges"], feats)
    assert int(got[0].nodes_per_graph.max()) >= 3000
    assert_rule(got, want)


# ---- errors ---------------------------------------------------------------------------------------------------------------
def _edit(path, fn):
    df = pd.read_csv(path, index_col=0, keep_default_na=False)
    fn(df).to_csv(path)


def _drop_graph_edges(df):
    return df[df.graph_id != df.graph_id.iloc[0]]


def _negative(df):
    df.loc[df.index[0], "innode"] = -1
    return df


def _dup(df):
    return pd.concat([df, df.iloc[:1]])


ERRORS = {
    "node_count": ("nodes.csv", lambda df: df.iloc[:-1], "node rows"),
    "no_edges": ("edges.csv", _drop_graph_edges, "no edge rows"),
    "negative": ("edges.csv", _negative, "negative endpoint"),
    "no_feature": (f"nodes_feat_{FEAT}_fixed.csv", lambda df: df.iloc[1:], "no feature row"),
    "duplicate": (f"nodes_feat_{FEAT}_fixed.csv", _dup, "more than one feature row"),
    "missing_column": ("nodes.csv", lambda df: df.drop(columns=["vuln"]), "no column 'vuln'"),
    "not_int": ("edges.csv", lambda df: df.assign(outnode=df.outnode.astype(object).where(df.index != df.index[3], "1e3")),
                r"edges.csv, line 5, column 'outnode': not an integer"),
}


@pytest.mark.parametrize("case", sorted(ERRORS) + ["unterminated"])
def test_errors_raise_value_error_and_free_device_memory(tmp_path, case):
    write_dataset(tmp_path, seed=3, n_graphs=30)
    folder = tmp_path / "bigvul"
    if case == "unterminated":
        with open(folder / "nodes.csv", "a") as f:
            f.write('999,"open\n')
        match = "nodes.csv, line .*: unterminated quote"
    else:
        name, fn, match = ERRORS[case]
        _edit(folder / name, fn)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    with pytest.raises(ValueError, match=match):
        IO.load_arena(tmp_path, DEV, feat=FEAT, concat_all_absdf=True)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) == before
