"""Cost of the encoder cache against the arena path over a frozen graph encoder, at the benchmark's C1 and C0 batches, with CUDA
events.

    python scripts/encoder_cache_cost.py [--rounds 5] [--steps 20] [--big-graphs 190000] [--out DIR]

Per size (C1: 1024 graphs x 150 nodes, C0: 256 graphs), over an arena of four batches' worth of graphs and a tensor-core module
(D = 128, T = 8, L = 2) with the embedding tables and the GatedGraphConv frozen, every configuration captured and replaying over
four rotating id lists of one shape, timed in alternating rounds of ``--steps`` calls each:
  * train_graph_arena / train_graph_cache:  FusedTrainer.step_ids(arena, ids) / step_ids(cache, ids), label_style="graph";
  * train_node_arena / train_node_cache:    the same in label_style="node" (every node a loss row);
  * eval_arena / eval_cache:                FusedEvaluator.update_ids(arena, ids) / update_ids(cache, ids);
  * cache_batch:                            ddfa_cache_batch alone, into the static outputs of one slot;
  * cache_batch_skewed:                     the same over lognormal graph sizes with one 3 000-node graph in the batch.
For each owner, the peak of ``torch.cuda.max_memory_allocated`` over its first call, above what was allocated before it — the
cache planes (``resident_cache_mib``) are allocated before, so a cache path holds them besides its first-call peak.  Then
the build time (host clock around EncoderCache(...) and a device synchronise), size and build peak of the cache of a
``--big-graphs``-graph synthetic arena of ~55-node graphs (0: skipped).  Prints one JSON line with the card's name, power limit
and SM clock, read in the same run (and writes it to DIR/encoder_cache_cost.json)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import synth  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
SIZES = {"C1": 1024, "C0": 256}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def frozen_module(style, dev):
    torch.manual_seed(0)
    m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, label_style=style, concat_all_absdf=True, positive_weight=2.0, engine="tcgen05").to(dev)
    for name, p in m.named_parameters():
        if not name.startswith(("output_layer.", "pooling.")):
            p.requires_grad_(False)
    return m


def first_call_peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def measure_size(B, args, dev):
    arena = D.GraphArena.from_graphs([synth.make_batch(4 * B, 150, seed=1)], dev)
    rng = np.random.default_rng(0)
    lists = [rng.choice(arena.num_graphs, B, replace=False) for _ in range(4)]
    turn = [0]

    def next_ids():
        turn[0] = (turn[0] + 1) % len(lists)
        return lists[turn[0]]

    calls, peak, keep = {}, {}, []
    for style in ("graph", "node"):
        for src in ("arena", "cache"):
            m = frozen_module(style, dev)
            tr = D.FusedTrainer(m, use_cuda_graph=True)
            s = arena if src == "arena" else D.EncoderCache(m, arena)     # after the trainer: the params live in its flat buffer
            fn = (lambda tr=tr, s=s: tr.step_ids(s, next_ids()))
            name = f"train_{style}_{src}"
            peak[name] = first_call_peak(fn)
            fn(); fn()                                                     # capture, replay
            calls[name] = fn
            keep.append((m, tr, s))
    m = frozen_module("graph", dev)
    cache = D.EncoderCache(m, arena)
    for src, s in (("arena", arena), ("cache", cache)):
        ev = D.FusedEvaluator(m)
        fn = (lambda ev=ev, s=s: ev.update_ids(s, next_ids()))
        peak[f"eval_{src}"] = first_call_peak(fn)
        fn(); fn()
        calls[f"eval_{src}"] = fn
        keep.append(ev)
    N = int(arena.nodes_per_graph[lists[0]].sum())
    # ddfa_cache_batch alone: over the fixed-size arena, and over one of lognormal graph sizes (mean 150 nodes) plus one
    # 3 000-node graph in every batch
    skew = D.GraphArena.from_graphs([synth.make_batch(4 * B, 150, seed=3, variable=True), synth.make_batch(1, 3000, seed=4)], dev)
    skew_cache = D.EncoderCache(m, skew)
    skew_ids = np.concatenate([rng.choice(4 * B, B - 1, replace=False), [4 * B]])
    sizes = {}
    for name, c, ids in (("cache_batch", cache, lists[0]), ("cache_batch_skewed", skew_cache, skew_ids)):
        n = int(c.arena.nodes_per_graph[ids].sum())
        out = c.alloc_outputs(B, n)
        out["ids"].copy_(torch.from_numpy(ids.astype(np.int32)))
        calls[name] = (lambda c=c, n=n, out=out: c._assemble(out["ids"], B, n, out))
        calls[name]()
        torch.cuda.synchronize()
        c._assemble(out["ids"], B, n, out).check()
        sizes[name] = (n, int(c.arena.nodes_per_graph[ids].max()), c.D)
        keep.append(out)
    times = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, fn in calls.items():
            times[k].append(timed(fn, args.steps))
    med = lambda xs: sorted(xs)[len(xs) // 2]                            # noqa: E731
    res = {"graphs": B, "nodes": N, "arena_graphs": arena.num_graphs,
           "resident_cache_mib": round(cache.nbytes / 2 ** 20, 1)}     # held besides every cache-path figure below
    for k in calls:
        res[k] = {"ms": [round(v, 4) for v in times[k]], "median_ms": round(med(times[k]), 4)}
        if k in peak:
            res[k]["first_call_peak_mib"] = round(peak[k] / 2 ** 20, 1)
    for what in ("train_graph", "train_node", "eval"):
        res[f"{what}_speedup"] = round(med(times[f"{what}_arena"]) / med(times[f"{what}_cache"]), 2)
    for name, (n, largest, d) in sizes.items():
        res[name]["nodes"], res[name]["largest_graph"] = n, largest
        res[name]["bytes_moved"] = 2 * (2 * n * d * 4) + 8 * n + 8 * B
        res[name]["gb_per_s"] = round(res[name]["bytes_moved"] / (med(times[name]) * 1e-3) / 1e9, 1)
    return res


def measure_build(G, dev):
    arena = D.GraphArena.from_graphs([synth.make_batch(G, 55, seed=2, variable=True)], dev)
    m = frozen_module("graph", dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    cache = D.EncoderCache(m, arena)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    return {"graphs": G, "nodes": cache.num_nodes, "D": cache.D, "build_s": round(seconds, 2), "cache_gb": round(cache.nbytes / 1e9, 2),
            "build_peak_above_arena_gb": round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--big-graphs", type=int, default=190_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_cache_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    result = {"card": card()}
    for name, B in SIZES.items():
        result[name] = measure_size(B, args, dev)
        torch.cuda.empty_cache()
    if args.big_graphs > 0:
        result["build"] = measure_build(args.big_graphs, dev)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "encoder_cache_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
