"""Cost of parameter groups / AdamW (FusedTrainer(param_groups=..., decoupled_weight_decay=True)) at the benchmark's C1 batch,
with CUDA events.

    python scripts/param_groups_cost.py [--rounds 10] [--steps 25]

Two single-GPU trainers on the same C1 batch (1024 graphs x 150 nodes, D = 128, T = 8, L = 2), both replaying captured steps:
the default (torch.optim.Adam, one group: ddfa_adam_flat_hp) and a two-group AdamW split as linevul_main.py builds it (biases
without weight decay: ddfa_adam_flat_groups).  They are timed in alternating rounds of ``--steps`` steps each.  Reports
milliseconds per step and the time of each trainer's Adam update alone (its update calls, launched eagerly).  Prints one JSON
line with the card's name and power limit, read in the same run."""
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
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("param_groups_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    batch = synth.make_batch(1024, 150, seed=11, variable=True, vuln_rate=0.3).to(dev)

    def trainer(grouped):
        torch.manual_seed(0)
        m = D.FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, 32, 8, 2, concat_all_absdf=True,
                                positive_weight=2.0, engine="tcgen05").to(dev)
        if not grouped:
            return D.FusedTrainer(m, use_cuda_graph=True)
        groups = [{"params": [p for n, p in m.named_parameters() if "bias" not in n], "weight_decay": 1e-2},
                  {"params": [p for n, p in m.named_parameters() if "bias" in n], "weight_decay": 0.0}]
        return D.FusedTrainer(m, use_cuda_graph=True, param_groups=groups, decoupled_weight_decay=True)
    trainers = {"adam": trainer(False), "adamw_2_groups": trainer(True)}
    for tr in trainers.values():
        for _ in range(3):                                       # eager warm-up, capture, replay
            tr.step(batch)
    torch.cuda.synchronize()
    per_step = {k: [] for k in trainers}
    for _ in range(args.rounds):
        for k, tr in trainers.items():
            per_step[k].append(timed(lambda: tr.step(batch), args.steps))
    adam_us = {}
    for k, tr in trainers.items():
        assert len(tr._graphs) == 1
        L, stream = _lib.lib(), torch.cuda.current_stream().cuda_stream

        def update():
            for name, a in tr._update:
                L.call(name, *a, stream)
        update()
        adam_us[k] = round(timed(update, 200) * 1e3, 2)
    med = lambda xs: sorted(xs)[len(xs) // 2]                    # noqa: E731
    print(json.dumps({"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "numel": trainers["adam"].numel,
                      "update_calls": {k: [n for n, _ in tr._update] for k, tr in trainers.items()},
                      "ms_per_step": {k: [round(x, 3) for x in v] for k, v in per_step.items()},
                      "median_ms_per_step": {k: round(med(v), 3) for k, v in per_step.items()},
                      "spread_ms_per_step": {k: round(max(v) - min(v), 3) for k, v in per_step.items()},
                      "adam_update_us_eager": adam_us}))


if __name__ == "__main__":
    main()
