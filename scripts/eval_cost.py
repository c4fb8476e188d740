"""Cost of an evaluation pass: FusedEvaluator against the module path, at the benchmark's C1 and C0 batches, with CUDA events.

    python scripts/eval_cost.py [--rounds 3] [--steps 10] [--out DIR]

For label_style "graph" and "node" (D = 128, T = 8, two output layers, tensor-core engine, positive_weight 2) and each batch
size (C1: 1024 graphs x ~150 nodes, C0: 256 graphs), three ways to evaluate the same pinned host batch, timed in alternating
rounds of ``--steps`` batches each:
  * host:   FusedEvaluator(use_cuda_graph=True).update(batch) with prefetch of the next batch (captured graph per shape);
  * ids:    FusedEvaluator.update_ids(arena, ids) over a GraphArena holding the same graphs;
  * module: module.validation_step((batch, {})) plus counting TP / FP / TN / FN on the host (what a Lightning loop feeding
            torchmetrics does per batch).
Every timed window ends with the metrics read on the host (``compute`` / the counts), so all three include their sync.  Also the
peak of ``torch.cuda.max_memory_allocated`` over the evaluator's first C1 batch, above what was allocated before it.  Prints one
JSON line with the card's name and power limit, read in the same run (and writes it to DIR/eval_cost.json)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import synth  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
SIZES = {"C1": 1024, "C0": 256}
ARMS = ("host", "ids", "module")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, finish, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    finish()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def module_arm(m, batch):
    acc = np.zeros(4, dtype=np.int64)

    def step():
        batch._cache.clear()          # a fresh batch every call, as in a validation loop: H2D copies and the CSR build each time
        _, p, y = m.validation_step((batch, {}))
        pred, t = p >= 0.5, y != 0
        acc[:] += [int((pred & t).sum()), int((pred & ~t).sum()), int((~pred & ~t).sum()), int((~pred & t).sum())]
    return step, lambda: None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    med = lambda xs: sorted(xs)[len(xs) // 2]                   # noqa: E731
    result = {"card": card(), "steps": args.steps, "rounds": args.rounds}
    for size, graphs in SIZES.items():
        for style in ("graph", "node"):
            torch.manual_seed(0)
            m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine="tcgen05",
                                    label_style=style).to(dev)
            batch = synth.make_batch(graphs, 150, seed=0, variable=True, vuln_rate=0.003 if style == "graph" else 0.06).pin_memory()
            arena = D.GraphArena.from_graphs([batch], device=dev)
            ids = np.arange(graphs)
            ev_host, ev_ids = D.FusedEvaluator(m), D.FusedEvaluator(m)
            row = {"graphs": graphs, "nodes": batch.num_nodes()}
            if size == "C1":
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                ev_host.update(batch)
                torch.cuda.synchronize()
                row["first_batch_peak_mib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)

            def host_step():
                ev_host.update(batch)
                ev_host.prefetch(batch)
            arms = {"host": (host_step, ev_host.compute), "ids": (lambda: ev_ids.update_ids(arena, ids), ev_ids.compute),
                    "module": module_arm(m, batch)}
            for _ in range(3):                                   # eager visit, capture, replay
                for a in ARMS:
                    arms[a][0]()
            times = {a: [] for a in ARMS}
            for _ in range(args.rounds):
                for a in ARMS:
                    times[a].append(timed(arms[a][0], arms[a][1], args.steps))
            for a in ARMS:
                ms = med(times[a])
                row[a] = {"ms": [round(v, 3) for v in times[a]], "median_ms": round(ms, 3), "graphs_per_s": round(graphs / ms * 1e3)}
            row["host_speedup_vs_module"] = round(med(times["module"]) / med(times["host"]), 2)
            ev_host.reset()
            ev_host.update(batch)
            f = ev_host.compute()
            row["val_confusion"] = f["val_confusion"]
            result[f"{size}_{style}"] = row
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "eval_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
