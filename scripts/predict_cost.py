"""Cost of scanning unlabeled functions: FusedPredictor against the module path, at the benchmark's C1 and C0 batches, and
ddfa_predict_store alone, with CUDA events.

    python scripts/predict_cost.py [--rounds 3] [--steps 10] [--out DIR]

Module: D = 128, T = 8, two output layers, tensor-core engine.  Per batch size (C1: 1024 graphs x ~150 nodes, C0: 256 graphs)
and configuration (graph style with statements None / "attention" / "saliency", node style with "probability", encoder_mode
with no statements; top_k = 10), timed in alternating rounds of ``--steps`` batches each:
  * host:   FusedPredictor.predict(batch) with prefetch of the next batch (captured graph per shape);
  * ids:    FusedPredictor.predict_ids(arena, ids) over a GraphArena holding the same graphs;
  * module: what a user writes without the predictor: module(batch, {}) under torch.no_grad() and torch.sigmoid, and in node
            style the function maximum (scatter_reduce) and a device-side stable sort per function (two stable torch.sort calls
            over the batch) for the top-k statements.  For graph style it runs once, against statements=None.
Every timed window ends with the results on the host side of a synchronise (``results()`` / torch.cuda.synchronize()).
``store``: ddfa_predict_store alone at the C1 shape (graph style, k = 10 over per-node scores) over 200 calls between two
events, and its share of the captured C1 batch with statements="attention" (host arm).  Prints one JSON line with the card's
name and power limit, read in the same run (and writes it to DIR/predict_cost.json)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200 import engine as E  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
SIZES = {"C1": 1024, "C0": 256}
CONFIGS = [("graph", None), ("graph", "attention"), ("graph", "saliency"), ("node", "probability"), ("encoder", None)]
TOP_K = 10


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


def module_arm(m, batch, node: bool, encoder: bool, dev):
    bnn = batch.batch_num_nodes().to(dev)
    B, N = batch.batch_size, batch.num_nodes()
    gid = torch.repeat_interleave(torch.arange(B, device=dev), bnn)
    start = torch.zeros(B, dtype=torch.int64, device=dev)
    start[1:] = torch.cumsum(bnn, 0)[:-1]
    pos = torch.arange(N, device=dev)

    def step():
        batch._cache.clear()          # a fresh batch every call, as in a scanning loop: H2D copies and the CSR build each time
        with torch.no_grad():
            out = m(batch, {})
        if encoder:
            return out
        p = torch.sigmoid(out)
        if node:
            prob = torch.zeros(B, device=dev).scatter_reduce(0, gid, p, "amax", include_self=False)
            o = torch.sort(p, descending=True, stable=True).indices
            o = o[torch.sort(gid[o], stable=True).indices]            # by function, score descending, node order among ties
            rank = pos - start[gid[o]]
            keep = rank < TOP_K
            top = torch.full((B, TOP_K), -1, dtype=torch.int64, device=dev)
            top[gid[o][keep], rank[keep]] = (o - start[gid[o]])[keep]
            return prob, top
        return p
    return step, torch.cuda.synchronize


def store_alone(dev, calls=200):
    """ddfa_predict_store at the C1 shape: 1024 functions of the synthetic batch's sizes, logits and per-node scores, k = 10."""
    b = synth.make_batch(1024, 150, seed=0, variable=True)
    bnn = b.batch_num_nodes().numpy()
    gptr = torch.from_numpy(np.concatenate([[0], np.cumsum(bnn)]).astype(np.int32)).to(dev)
    N, B = int(bnn.sum()), len(bnn)
    g = torch.Generator(device=dev).manual_seed(0)
    scores = torch.rand(N, device=dev, generator=g)
    logits = torch.randn(B, device=dev, generator=g)
    C = B * (calls + 10)
    prob = torch.empty(C, device=dev)
    idx = torch.empty(C, TOP_K, dtype=torch.int32, device=dev)
    top = torch.empty(C, TOP_K, device=dev)
    cursor = torch.zeros(2, dtype=torch.int64, device=dev)
    L = _lib.lib()

    def call():
        L.call("ddfa_predict_store", logits.data_ptr(), None, None, 0, scores.data_ptr(), TOP_K, gptr.data_ptr(), B, B, prob.data_ptr(),
               None, idx.data_ptr(), top.data_ptr(), cursor.data_ptr(), C, E._stream_ptr())
    for _ in range(5):
        call()
    cursor.zero_()
    return timed(call, lambda: None, calls), N


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("predict_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    med = lambda xs: sorted(xs)[len(xs) // 2]                   # noqa: E731
    result = {"card": card(), "steps": args.steps, "rounds": args.rounds, "top_k": TOP_K}
    for size, graphs in SIZES.items():
        for style, statements in CONFIGS:
            torch.manual_seed(0)
            encoder = style == "encoder"
            m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, engine="tcgen05", encoder_mode=encoder,
                                    label_style="node" if style == "node" else "graph").to(dev)
            batch = synth.make_batch(graphs, 150, seed=0, variable=True).pin_memory()
            arena = D.GraphArena.from_graphs([batch], device=dev)
            ids = np.arange(graphs)
            cap = graphs * (args.steps + 4)
            kw = {"statements": statements, "top_k": TOP_K} if statements else {}
            pr_host, pr_ids = D.FusedPredictor(m, capacity=cap, **kw), D.FusedPredictor(m, capacity=cap, **kw)

            def host_step():
                pr_host.predict(batch)
                pr_host.prefetch(batch)
            arms = {"host": (host_step, pr_host.results, pr_host.reset), "ids": (lambda: pr_ids.predict_ids(arena, ids), pr_ids.results,
                                                                                 pr_ids.reset)}
            if statements in (None, "probability"):
                step, finish = module_arm(m, batch, style == "node", encoder, dev)
                arms["module"] = (step, finish, lambda: None)
            for _ in range(3):                                   # eager visit, capture, replay
                for a in arms:
                    arms[a][0]()
            times = {a: [] for a in arms}
            for _ in range(args.rounds):
                for a in arms:
                    arms[a][2]()
                    times[a].append(timed(arms[a][0], arms[a][1], args.steps))
            row = {"graphs": graphs, "nodes": batch.num_nodes()}
            for a in arms:
                ms = med(times[a])
                row[a] = {"ms": [round(v, 3) for v in times[a]], "median_ms": round(ms, 3), "graphs_per_s": round(graphs / ms * 1e3)}
            if "module" in arms:
                row["host_speedup_vs_module"] = round(med(times["module"]) / med(times["host"]), 2)
            result[f"{size}_{style}_{statements or 'none'}"] = row
    store_ms, n = store_alone(dev)
    c1 = result["C1_graph_attention"]["host"]["median_ms"]
    result["store"] = {"functions": 1024, "nodes": n, "us_per_call": round(store_ms * 1e3, 2),
                       "share_of_C1_attention_batch_pct": round(100 * store_ms / c1, 3)}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "predict_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
