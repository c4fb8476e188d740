"""Cost of the gradient guard (FusedTrainer(max_grad_norm=..., skip_nonfinite=...)) at the benchmark's C1 batch, with CUDA events.

    python scripts/grad_guard_cost.py [--rounds 10] [--steps 100]

Two single-GPU trainers on the same C1 batch (1024 graphs x 150 nodes, D = 128, T = 8, L = 2), both replaying a captured step:
one without the guard, one with skip_nonfinite and a bound that clips every step.  They are timed in alternating rounds of
``--steps`` replays each.  Also times ddfa_grad_norm alone on the flat gradient buffer.  Prints one JSON line with the card's name
and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import _lib, synth  # noqa: E402


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
    return a.elapsed_time(b) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_guard_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    batch = synth.make_batch(1024, 150, seed=11, variable=True, vuln_rate=0.3).to(dev)

    def trainer(**kw):
        torch.manual_seed(0)
        m = D.FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, 32, 8, 2, concat_all_absdf=True,
                                positive_weight=2.0, engine="tcgen05").to(dev)
        return D.FusedTrainer(m, use_cuda_graph=True, **kw)
    off = trainer()
    on = trainer(max_grad_norm=1e-3, skip_nonfinite=True)      # far below the C1 gradient norm: every step clips
    for tr in (off, on):
        for _ in range(3):                                      # eager warm-up, capture, replay
            tr.step(batch)
    torch.cuda.synchronize()
    clipped = float(on.grad_norm) > on.max_grad_norm
    t_off, t_on = [], []
    for _ in range(args.rounds):
        t_off.append(timed(lambda: off.step(batch), args.steps))
        t_on.append(timed(lambda: on.step(batch), args.steps))
    L = _lib.lib()
    ws = torch.empty(L.call("ddfa_grad_norm_workspace_bytes", on.numel), dtype=torch.uint8, device=dev)
    gstate = torch.zeros(4, device=dev)

    def norm():      # on the current stream: the capture below records on a stream of its own
        L.call("ddfa_grad_norm", on.flat_g.data_ptr(), on.numel, on._max_norm_dev.data_ptr(), gstate.data_ptr(), ws.data_ptr(), ws.numel(),
               torch.cuda.current_stream().cuda_stream)
    norm()
    norm_us = timed(norm, 200)
    g = torch.cuda.CUDAGraph()                                  # launch overhead as a captured step sees it
    with torch.cuda.graph(g):
        for _ in range(20):
            norm()
    g.replay()
    torch.cuda.synchronize()
    norm_graph_us = timed(g.replay, 20) / 20
    med = lambda xs: sorted(xs)[len(xs) // 2]                   # noqa: E731
    print(json.dumps({"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "numel": on.numel,
                      "every_step_clips": clipped, "skipped_steps": on.skipped_steps,
                      "step_us_guard_off": [round(x, 1) for x in t_off], "step_us_guard_on": [round(x, 1) for x in t_on],
                      "median_delta_us": round(med(t_on) - med(t_off), 1),
                      "median_delta_pct": round(100 * (med(t_on) - med(t_off)) / med(t_off), 2),
                      "grad_norm_us_eager": round(norm_us, 2), "grad_norm_us_in_graph": round(norm_graph_us, 2)}))


if __name__ == "__main__":
    main()
