"""The CSV rules of the device loader (tests/csv_rule.py) against pandas.read_csv, the parser bigvul_io's host path uses, on
text that to_csv writes for awkward ``code`` strings, line ends, blank lines, header orders and integral floats."""
import io
import os
import sys

import numpy as np
import pandas as pd
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import csv_rule as R  # noqa: E402

AWKWARD = ["a, b", 'say "hi"', '""', "line1\nline2", "crlf\r\nnext", "", "nan", "NaN", "é → ü 中文", ",", '"', "\n", "x\r\n\r\ny",
           "trailing,", 'q","r']


def awkward_frame(rng, rows, extra=False):
    df = pd.DataFrame({
        "dgl_id": np.arange(rows),
        "code": [AWKWARD[i] for i in rng.integers(0, len(AWKWARD), rows)],
        "vuln": rng.integers(0, 2, rows),
        "graph_id": rng.integers(-5, 10 ** 12, rows),
        "node_id": rng.integers(0, 2 ** 40, rows),
    })
    if extra:
        df["lineNumber"] = rng.random(rows)
        df["_label"] = "CALL"
    return df


def rows_of(text: bytes, names):
    spans, data = R.row_spans(text)
    header = [R.unquote(f) for f in R.split_fields(data[spans[0][0]:spans[0][1]])]
    pos = [header.index(n) for n in names]
    return [[R.unquote(R.split_fields(data[s:e])[p]) for p in pos] for s, e in spans[1:]]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("lineterminator", ["\n", "\r\n"])
def test_rows_and_fields_match_read_csv(seed, lineterminator):
    rng = np.random.default_rng(seed)
    df = awkward_frame(rng, 300, extra=seed % 2 == 1)
    cols = list(df.columns)
    rng.shuffle(cols)                                  # permuted header
    text = df[cols].to_csv(lineterminator=lineterminator).encode("utf-8")
    ref = pd.read_csv(io.BytesIO(text), index_col=0, keep_default_na=False, dtype={"code": str})
    got = R.read_columns(text, ["graph_id", "node_id", "vuln", "dgl_id"])
    for name in got:
        assert got[name].tolist() == ref[name].tolist(), name
    assert [r[0] for r in rows_of(text, ["code"])] == ref["code"].tolist()


def test_blank_lines_and_no_final_newline():
    text = b'\n\n,graph_id,code,node_id\r\n\r\n0,3,"a\n\nb",7\n\n\n1,-4,"x,""y""",8\r\n2,5,,9'
    ref = pd.read_csv(io.BytesIO(text), index_col=0, keep_default_na=False)
    got = R.read_columns(text, ["graph_id", "node_id"])
    assert got["graph_id"].tolist() == ref["graph_id"].tolist() == [3, -4, 5]
    assert got["node_id"].tolist() == ref["node_id"].tolist() == [7, 8, 9]
    assert [r[0] for r in rows_of(text, ["code"])] == ref["code"].tolist()


def test_integral_floats_and_bad_tokens():
    text = b",graph_id,v\n0,1,5.0\n1,2,-3.00\n2,3,\"7\"\n3,4,8.\n"
    ref = pd.read_csv(io.BytesIO(text), index_col=0)
    got = R.read_columns(text, ["graph_id", "v"])
    assert got["v"].tolist() == [int(x) for x in ref["v"].tolist()] == [5, -3, 7, 8]
    for bad in (b"5.5", b"1e3", b"", b"nan", b" 4", b"x", b"9223372036854775808", b"--1"):
        with pytest.raises(ValueError) as e:
            R.read_columns(b",graph_id,v\n0,1,2\n1,2," + bad + b"\n", ["graph_id", "v"])
        assert e.value.args == (3, "v")
    assert R.to_int(b"-9223372036854775808") == -2 ** 63 and R.to_int(b"9223372036854775807") == 2 ** 63 - 1

