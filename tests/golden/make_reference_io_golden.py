"""Pins deepdfa_b200/bigvul_io.py against the reference's own data-loading code — by running that code.

Runs, from <reference root>/DDFA (first argument), on the synthetic processed-dataset files of tests/bigvul_fixture.py:

    sastvd/linevd/graphmogrifier.py   get_nodes_df (:20-40), get_graphs (:59-95)      the REAL functions
    sastvd/helpers/dclass.py          BigVulDataset.get_epoch_indices (:84-105)       the REAL method (on a stand-in `self`)

Stand-ins: `dgl` is not installed, so `graphmogrifier.get_graphs_by_id` (which only does `dgl.data.utils.load_graphs` of the
graphs.bin that dbize_graphs.py wrote from edges.csv) is replaced by deepdfa_b200.bigvul_io.read_edge_graphs on the same
edges.csv — the edge-list semantics therefore stay a restatement (dbize_graphs.py:17-27 is three lines of DGL calls) — and
`sastvd.helpers.datasets` / `.joern` (unused on this path, they import unidiff etc.) are empty modules.  `SINGSTORAGE`
points the reference's `processed_dir()` at the temporary dataset.

Run in the build container:   python tests/golden/make_reference_io_golden.py
Writes tests/golden/reference_io_golden.pt; tests/test_bigvul_io.py::test_reader_matches_reference_loaders reads it.
"""
import os
import sys
import tempfile
import types
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REFERENCE = os.path.join(sys.argv[1] if len(sys.argv) > 1 else ".", "DDFA")

from bigvul_fixture import FEAT, write_dataset  # noqa: E402
from deepdfa_b200 import bigvul_io as IO  # noqa: E402


def main():
    tmp = Path(tempfile.mkdtemp())
    os.environ["SINGSTORAGE"] = str(tmp)                       # sastvd.storage_dir() = $SINGSTORAGE/storage
    processed = tmp / "storage" / "processed"
    write_dataset(processed, seed=0, n_graphs=7)

    for n in ("sastvd.helpers.datasets", "sastvd.helpers.joern"):
        sys.modules[n] = types.ModuleType(n)
    dgl = types.ModuleType("dgl")
    dgl.data = types.ModuleType("dgl.data")
    dgl.data.utils = types.ModuleType("dgl.data.utils")
    dgl.data.utils.load_graphs = None
    dgl.HeteroGraph = object
    sys.modules.update({"dgl": dgl, "dgl.data": dgl.data, "dgl.data.utils": dgl.data.utils})
    sys.path.insert(0, REFERENCE)
    import sastvd.linevd.graphmogrifier as gm                     # the real module
    import sastvd.helpers.dclass as dc

    # graphs.bin stand-in: the graphs dbize_graphs.py would have saved, built from the same edges.csv
    gm.get_graphs_by_id = lambda dsname, sample_mode: IO.read_edge_graphs(processed / dsname / "edges.csv")

    nodes_df = gm.get_nodes_df("bigvul", False, FEAT, concat_all_absdf=True)
    graphs_by_id, extrafeats = gm.get_graphs("bigvul", nodes_df, False, FEAT, "train", True, True)
    golden = {
        "nodes_columns": list(nodes_df.columns),
        "nodes_records": nodes_df.drop(columns=["code", "_label"]).to_dict(orient="list"),
        "graph_ids": [int(k) for k in graphs_by_id],
        "ndata": {int(k): {name: v.clone() for name, v in g.ndata.items()} for k, g in graphs_by_id.items()},
        "num_nodes": {int(k): g.num_nodes() for k, g in graphs_by_id.items()},
    }

    rng0 = np.random.default_rng(3)
    df = pd.DataFrame({"id": np.arange(500) * 7, "vul": (rng0.random(500) < 0.12).astype(int)})
    epochs = {}
    for undersample, oversample in (("v1.0", None), ("v2.5", None), (0.25, None), (None, 2.0), ("v1.0", 1.5), (None, None)):
        me = SimpleNamespace(df=df, undersample=undersample, oversample=oversample, rng=np.random.RandomState(0))
        epochs[f"{undersample}|{oversample}"] = [list(map(int, dc.BigVulDataset.get_epoch_indices(me))) for _ in range(3)]
    golden["epoch_indices"] = epochs
    out = os.path.join(ROOT, "tests", "golden", "reference_io_golden.pt")
    torch.save(golden, out)
    print("wrote", out, len(golden["graph_ids"]), "graphs;", {k: len(v[0]) for k, v in epochs.items()})


if __name__ == "__main__":
    main()
