"""Cost of the DeepLift, DeepLiftShap and GradientShap statement scores in FusedEvaluator: ms per captured batch and the peak memory
of the first batch for each mode, next to the plain evaluator batch, saliency and integrated gradients at m = 16.  C1 (1024 graphs)
and C0 (256 graphs) synthetic batches, tcgen05 engine, hidden width 128, T = 5, three head layers.  Prints one JSON line per
measurement, with the card's name and power limit.

    python scripts/attribution_cost.py [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import synth  # noqa: E402

DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
# (statements, evaluator arguments)
MODES = [(None, {}), ("saliency", {}), ("integrated_gradients", dict(ig_steps=16)), ("deeplift", {}),
         ("deeplift_shap", {}), ("deeplift_shap", dict(baseline_stdev=0.1)), ("gradient_shap", {}),
         ("gradient_shap", dict(baseline_stdev=0.1, noise_stdev=0.1))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    gpu = card()
    torch.manual_seed(0)
    m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 5, 3, concat_all_absdf=True, engine="tcgen05").to(DEV)
    out = open(args.out, "a") if args.out else None
    for name, graphs in (("C1", 1024), ("C0", 256)):
        b = synth.make_batch(graphs, 150, seed=1, variable=True, vuln_rate=0.3)
        base = None
        for mode, kw in MODES:
            ev = D.FusedEvaluator(m, statements=mode, **kw)
            heavy = mode in ("integrated_gradients", "gradient_shap") or ev.shap_samples > 1 and mode == "deeplift_shap" \
                and ev.baseline_stdev > 0
            reps = max(3, args.reps // (4 if heavy else 1))
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            mem0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            ev.update(b)                    # the first (eager) visit: workspace growth
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - mem0
            ev.update(b)                    # capture
            ms = timed(lambda: ev.update(b), reps)
            base = ms if mode is None else base
            line = json.dumps({"batch": name, "nodes": b.num_nodes(), "statements": mode, **kw,
                               "samples": ev.shap_samples if mode in ("deeplift_shap", "gradient_shap") else None,
                               "ms_per_batch_captured": round(ms, 3), "x_plain": round(ms / base, 2),
                               "first_batch_peak_mib": round(peak / 2 ** 20, 1), "gpu": gpu})
            print(line, flush=True)
            if out:
                out.write(line + "\n")
                out.flush()
            del ev


if __name__ == "__main__":
    main()
