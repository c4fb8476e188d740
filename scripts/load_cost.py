"""Cost of building the arena from the processed Big-Vul files: bigvul_io.load_arena (on the device, csrc/csv_load.cu) against
the host composition GraphArena.from_graphs([load_graphs(...)[i] ...]) at 20 000 graphs, and load_arena alone at Big-Vul
size (190 000 graphs, lognormal sizes, > 10 M nodes).  Files are generated in a temporary directory (deleted afterwards) by
synth.write_bigvul_files; they have just been written, so they are read from the page cache.

Reported per set: file bytes; load_arena wall time (median of --repeats, each ending in a device sync) split into file read
into pinned memory, H2D copy, row index + field parse, and the rest (sorts, grouping, union COO, joins, CSR build, arena);
bytes parsed per second; peak device memory of one call; the host composition's time where it runs; the card name and power
limit read in the same run.

    python scripts/load_cost.py [--graphs 190000] [--small 20000] [--repeats 3] [--out results.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepdfa_b200 import bigvul_io as IO, synth  # noqa: E402
from deepdfa_b200.arena import GraphArena  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "not read"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def phases(root, feat):
    """Read, H2D and parse time per file, with the columns load_arena reads from it."""
    loader = IO._DeviceLoad(root, DEV, "bigvul", feat, True, False)
    folder = Path(root) / "bigvul"
    files = [(folder / "nodes.csv", [("graph_id", False), ("node_id", False), ("vuln", False)]),
             (folder / "edges.csv", [("graph_id", False), ("innode", False), ("outnode", False)])]
    for path in sorted({p for _, p, _, _ in loader.features}):
        files.append((path, [("graph_id", False), ("node_id", False), ("_ABS_DATAFLOW", True)]))
    read = h2d = parse = 0.0
    for path, cols in files:
        size = path.stat().st_size
        host = torch.empty(size, dtype=torch.uint8, pin_memory=True)
        t0 = time.perf_counter()
        with open(path, "rb") as f:
            f.readinto(memoryview(host.numpy()))
        read += time.perf_counter() - t0
        dev = torch.empty(size, dtype=torch.uint8, device=DEV)
        _, t = timed(lambda: dev.copy_(host, non_blocking=True))
        h2d += t
        del dev, host
        _, t = timed(lambda: loader._parse(path, cols))
        parse += t
    parse -= read + h2d                      # _parse reads and copies too
    return read, h2d, parse


def measure(root, feat, repeats, host_path):
    total_bytes = sum(p.stat().st_size for p in (Path(root) / "bigvul").iterdir())
    kw = dict(feat=feat, concat_all_absdf=True)
    IO.load_arena(root, DEV, **kw)           # warm-up: module load, allocator
    times = []
    for _ in range(repeats):
        torch.cuda.reset_peak_memory_stats(DEV)
        base = torch.cuda.memory_allocated(DEV)
        (arena, ids), t = timed(lambda: IO.load_arena(root, DEV, **kw))
        times.append(t)
        peak = torch.cuda.max_memory_allocated(DEV) - base
        arena_bytes = sum(x.numel() * x.element_size() for x in [arena.dg.indptr, arena.dg.indices, arena.dg.indptr_t,
                                                                   arena.dg.indices_t, arena.dg.graph_ptr, arena.node_off, arena.vuln,
                                                                   *arena.feats.values()])
        del arena, ids
    total = float(np.median(times))
    read, h2d, parse = phases(root, feat)
    out = {"file_bytes": total_bytes, "load_arena_s": total, "load_arena_s_all": times, "read_s": read, "h2d_s": h2d,
           "parse_s": parse, "group_join_csr_s": total - read - h2d - parse, "bytes_per_s": total_bytes / total,
           "peak_device_bytes": int(peak), "arena_bytes": int(arena_bytes), "files_in_page_cache": "yes (just written)"}
    if host_path:
        def host():
            graphs = IO.load_graphs(root, "bigvul", **kw)
            return GraphArena.from_graphs([graphs[i] for i in sorted(graphs)], DEV)
        _, out["host_composition_s"] = timed(host)
    else:
        out["host_composition_s"] = "not measured"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=190_000)
    ap.add_argument("--small", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "load_cost.py needs a GPU"
    feat = f"_ABS_DATAFLOW_datatype{synth.BIGVUL_TAIL}"
    result = {"card": card()}
    for name, n, host_path in (("small", a.small, True), ("bigvul", a.graphs, False)):
        root = Path(tempfile.mkdtemp())
        try:
            t = synth.write_bigvul_files(root, n, seed=1)
            r = measure(root, feat, a.repeats, host_path)
            r.update(graphs=n, nodes=int(t["nodes"]["graph_id"].shape[0]), edge_rows=int(t["edges"]["graph_id"].shape[0]))
            result[name] = r
            print(name, json.dumps(r), flush=True)
        finally:
            shutil.rmtree(root, ignore_errors=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(result, indent=1))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
