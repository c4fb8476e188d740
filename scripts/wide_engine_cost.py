"""Cost of the tensor-core engine at the wide widths (csrc/gru_tc_wide.cu) against the SIMT engine, at the benchmark's C1 batch,
with CUDA events.

    python scripts/wide_engine_cost.py [--rounds 6] [--steps 10] [--widths 256 512]

For each width W (hidden_dim W / 4 with concat_all_absdf, T = 8, two output layers) two single-GPU trainers on the same C1 batch
(1024 graphs x 150 nodes) replay captured steps, engine="simt" and engine="tcgen05", timed in alternating rounds of ``--steps``
steps each.  Then each of the step's GEMM shapes on its own (N = the batch's node count): ddfa_sgemm for SIMT and
ddfa_gru_tc_wide_gemm for the tensor cores (which includes turning its fp32 operands into bf16 hi / lo images), with the
achieved TFLOP/s 2 M N K / time (the useful products, not the three bf16 products per term).  Prints one JSON line with the
card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200.engine import _p  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


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


def gemm_costs(N, W, iters):
    """ms and TFLOP/s of the step's GEMM shapes on both engines (the weight gradient accumulates, as in the step)."""
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    dev = "cuda:0"
    s, w = torch.randn(N, W, device=dev), torch.randn(3 * W, W, device=dev) * W ** -0.5
    q, out_f, out_d = torch.randn(N, 3 * W, device=dev), torch.empty(N, 3 * W, device=dev), torch.zeros(N, W, device=dev)
    dw = torch.zeros(3 * W, W, device=dev)
    tiles = -(-3 * W // 128) * -(-W // 128)
    split = max(1, min((2 * 132 + tiles - 1) // tiles, (N + 15) // 16 // 8))      # gru_step.cu: simt_wgrad_split
    simt = {"fwd": lambda: L.call("ddfa_sgemm", 0, 1, N, 3 * W, W, 1.0, _p(s), W, _p(w), W, 0.0, _p(out_f), 3 * W, 1, st),
            "dgrad": lambda: L.call("ddfa_sgemm", 0, 0, N, W, 3 * W, 1.0, _p(q), 3 * W, _p(w), W, 0.0, _p(out_d), W, 1, st),
            "wgrad": lambda: L.call("ddfa_sgemm", 1, 0, 3 * W, W, N, 1.0, _p(q), 3 * W, _p(s), W, 1.0, _p(dw), W, split, st)}
    calls = {"fwd": (0, s, w, out_f), "dgrad": (1, q, w, out_d), "wgrad": (3, q, s, dw)}
    wsb = max(L.call("ddfa_gru_tc_wide_gemm_workspace_bytes", c, N, W) for c, *_ in calls.values())
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    tc = {k: (lambda c=c, a=a, b=b, o=o: L.call("ddfa_gru_tc_wide_gemm", c, _p(a), _p(b), N, W, _p(o), _p(ws), wsb, st))
          for k, (c, a, b, o) in calls.items()}
    flops = 2.0 * N * 3 * W * W          # every shape: M N K = N x 3W x W
    out = {}
    for name in ("fwd", "dgrad", "wgrad"):
        for eng, fns in (("simt", simt), ("tcgen05", tc)):
            fns[name]()
            ms = timed(fns[name], iters)
            out[f"{eng} {name}"] = {"ms": round(ms, 3), "tflops": round(flops / ms / 1e9, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--widths", type=int, nargs="+", default=[256, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_engine_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    batch = synth.make_batch(1024, 150, seed=11, variable=True, vuln_rate=0.3).to(dev)
    result = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "nodes": batch.num_nodes(), "widths": {}}
    for W in args.widths:
        trainers = {}
        for engine in ("simt", "tcgen05"):
            torch.manual_seed(0)
            m = D.FlowGNNGGNNModule(FEAT, 1002, W // 4, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine).to(dev)
            trainers[engine] = D.FusedTrainer(m, use_cuda_graph=True)
        for tr in trainers.values():
            for _ in range(3):                                   # eager warm-up, capture, replay
                tr.step(batch)
        torch.cuda.synchronize()
        per_step = {k: [] for k in trainers}
        for _ in range(args.rounds):
            for k, tr in trainers.items():
                per_step[k].append(timed(lambda: tr.step(batch), args.steps))
        del trainers
        torch.cuda.empty_cache()
        med = lambda xs: sorted(xs)[len(xs) // 2]                # noqa: E731
        result["widths"][W] = {"ms_per_step": {k: [round(x, 2) for x in v] for k, v in per_step.items()},
                               "median_ms_per_step": {k: round(med(v), 2) for k, v in per_step.items()},
                               "speedup": round(med(per_step["simt"]) / med(per_step["tcgen05"]), 2),
                               "gemms": gemm_costs(batch.num_nodes(), W, 20)}
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
