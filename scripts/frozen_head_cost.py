"""Cost of a FusedTrainer step with frozen parameters at the benchmark's C1 batch, with CUDA events.

    python scripts/frozen_head_cost.py [--rounds 5] [--steps 20] [--out DIR]

Three configurations of the same graph-style module (1024 graphs x 150 nodes, D = 128, T = 8, L = 2, tensor-core engine), each
a FusedTrainer(use_cuda_graph=True) replaying its captured step on one resident batch, timed in alternating rounds of
``--steps`` steps each:
  * all:     every parameter trainable (the step the benchmark times);
  * tables:  the four embedding tables frozen (full GGNN backward, no embedding backward);
  * encoder: tables and GatedGraphConv frozen, the readout gate and the MLP head trained (main_cli.py --freeze_graph): the GGNN
             runs in its inference form and the backward stops after the readout.
For each, the peak of ``torch.cuda.max_memory_allocated`` over its first step, above what was allocated before that step.
Prints one JSON line with the card's name and power limit, read in the same run (and writes it to DIR/frozen_head_cost.json)."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import synth  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
CONFIGS = ("all", "tables", "encoder")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
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


def trainer(config, dev):
    torch.manual_seed(0)
    m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine="tcgen05").to(dev)
    for name, p in m.named_parameters():
        head = name.startswith(("output_layer.", "pooling."))
        if (config == "tables" and "embedding" in name) or (config == "encoder" and not head):
            p.requires_grad_(False)
    return D.FusedTrainer(m, use_cuda_graph=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frozen_head_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    batch = synth.make_batch(1024, 150, seed=0).to(dev)
    med = lambda xs: sorted(xs)[len(xs) // 2]                   # noqa: E731
    result = {"card": card(), "graphs": batch.batch_size, "nodes": batch.num_nodes(), "edges": batch.num_edges()}
    trainers, peak = {}, {}
    for c in CONFIGS:
        tr = trainer(c, dev)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        tr.step(batch)                                          # eager: grows the workspace
        torch.cuda.synchronize()
        peak[c] = torch.cuda.max_memory_allocated() - base
        for _ in range(2):                                      # capture, replay
            tr.step(batch)
        trainers[c] = tr
    times = {c: [] for c in CONFIGS}
    for _ in range(args.rounds):
        for c in CONFIGS:
            times[c].append(timed(lambda: trainers[c].step(batch), args.steps))
    for c in CONFIGS:
        result[c] = {"ms": [round(v, 3) for v in times[c]], "median_ms": round(med(times[c]), 3),
                     "step_peak_mib": round(peak[c] / 2 ** 20, 1)}
    for c in CONFIGS[1:]:
        result[c]["speedup_vs_all"] = round(med(times["all"]) / med(times[c]), 2)
        result[c]["peak_share_of_all"] = round(peak[c] / peak["all"], 3)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frozen_head_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
