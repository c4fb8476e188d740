"""Cost of statement-level localisation in FusedEvaluator: ms per captured batch for each statements= mode against the plain
evaluator batch, integrated gradients at m = 16 and 50, the peak memory of the first batch, and the dgrad-only backward
(engine.backward(grad_weights=False)) against the full one.  C1 (1024 graphs) and C0 (256 graphs) synthetic batches, tcgen05
engine, hidden width 128.  Prints one JSON line per measurement, with the card's name and power limit.

    python scripts/statements_cost.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import engine as E, synth  # noqa: E402
from deepdfa_b200.module import _ENGINES  # noqa: E402

DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


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
    args = ap.parse_args()
    gpu = card()
    torch.manual_seed(0)
    m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 5, 3, concat_all_absdf=True, engine="tcgen05").to(DEV)
    for name, graphs in (("C1", 1024), ("C0", 256)):
        b = synth.make_batch(graphs, 150, seed=1, variable=True, vuln_rate=0.3)
        base = None
        for mode, steps in ((None, 0), ("attention", 0), ("saliency", 0), ("integrated_gradients", 16), ("integrated_gradients", 50)):
            reps = max(3, args.reps // (10 if steps == 50 else 1))
            ev = D.FusedEvaluator(m, statements=mode, ig_steps=max(steps, 1))
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
            print(json.dumps({"batch": name, "nodes": b.num_nodes(), "statements": mode, "ig_steps": steps or None,
                              "ms_per_batch_captured": round(ms, 3), "x_plain": round(ms / base, 2),
                              "first_batch_peak_mib": round(peak / 2 ** 20, 1), "gpu": gpu}), flush=True)
            del ev
        # the backward alone, eager: full (weight gradients into a scratch pack) against dgrad-only
        dg = E.prepare_graph(b, DEV)
        idx = E.node_indices(b, True, FEAT, DEV)
        params = E.ParamPack.from_flat_list([p.data for p in m.param_list()], len(m._tables()), m._num_layers)
        grads = params.zeros_like()
        ws = E.Workspace(torch.device(DEV))
        eng = _ENGINES[m.engine]
        _, _, saved = E.forward(params, dg, idx, 5, training=True, engine=eng, alloc=ws)
        ones = torch.ones(b.batch_size, device=DEV)
        res = {}
        for gw in (True, False):
            res[gw] = timed(lambda: E.backward(params, dg, saved, grads, dlogits=ones, engine=eng, alloc=ws, grad_weights=gw), args.reps)
        print(json.dumps({"batch": name, "backward_full_ms": round(res[True], 3), "backward_dgrad_only_ms": round(res[False], 3),
                          "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
