"""Cost of gradient accumulation (FusedTrainer(accumulate_grad_batches=k)) at the benchmark's C1 batch, with CUDA events.

    python scripts/accumulate_cost.py [--rounds 10] [--windows 25]

Two single-GPU trainers on the same C1 batch (1024 graphs x 150 nodes, D = 128, T = 8, L = 2), both replaying captured steps:
one with k = 1 and one with k = 4.  They are timed in alternating rounds of ``--windows`` windows each (k = 1: one step per
window; k = 4: four micro-batches, three accumulating and one applying).  Reports milliseconds per micro-batch and per window,
and times ddfa_grad_accumulate alone over the flat gradient buffer.  Prints one JSON line with the card's name and power limit,
read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200 import engine as E  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--windows", type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("accumulate_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    batch = synth.make_batch(1024, 150, seed=11, variable=True, vuln_rate=0.3).to(dev)

    def trainer(k):
        torch.manual_seed(0)
        m = D.FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, 32, 8, 2, concat_all_absdf=True,
                                positive_weight=2.0, engine="tcgen05").to(dev)
        return D.FusedTrainer(m, use_cuda_graph=True, accumulate_grad_batches=k)
    trainers = {1: trainer(1), 4: trainer(4)}
    for k, tr in trainers.items():
        for _ in range(3 * k):                                   # every phase: eager warm-up, capture, replay
            tr.step(batch)
    torch.cuda.synchronize()
    per_window = {1: [], 4: []}
    for _ in range(args.rounds):
        for k, tr in trainers.items():
            per_window[k].append(timed(lambda: [tr.step(batch) for _ in range(k)], args.windows))
    tr = trainers[4]
    assert tr.accumulated == 0 and len(tr._graphs) == 3 and len(trainers[1]._graphs) == 1    # first / add / apply; one step
    acc = torch.zeros(tr.numel, device=dev)

    def add():
        E.grad_accumulate(acc, tr.flat_g, 0, tr.numel, _lib.GRAD_ACC_ADD)
    add()
    add_us = timed(add, 200) * 1e3
    med = lambda xs: sorted(xs)[len(xs) // 2]                    # noqa: E731
    print(json.dumps({"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "numel": tr.numel,
                      "captured_graphs_k1": len(trainers[1]._graphs), "captured_graphs_k4": len(tr._graphs),
                      "ms_per_window_k1": [round(x, 3) for x in per_window[1]],
                      "ms_per_window_k4": [round(x, 3) for x in per_window[4]],
                      "median_ms_per_micro_batch_k1": round(med(per_window[1]), 3),
                      "median_ms_per_micro_batch_k4": round(med(per_window[4]) / 4, 3),
                      "median_ms_per_window_k1": round(med(per_window[1]), 3),
                      "median_ms_per_window_k4": round(med(per_window[4]), 3),
                      "grad_accumulate_us_eager": round(add_us, 2)}))


if __name__ == "__main__":
    main()
