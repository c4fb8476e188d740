"""Cost of the test pass's threshold curves: binary_curves on the device against the host path it replaces (copy the
predictions to the host, sort them with NumPy, apply the same torchmetrics < 0.10 rules there).

    python scripts/curve_cost.py [--rounds 5] [--out DIR]

Sizes at a 6 % positive rate: 19 000 samples (a graph-style Big-Vul test split), 10^6 (a node-style split) and 10.4 M (every
statement of the arena).  Per size, in alternating rounds after one warm-up call of each:
  * device: binary_curves(probs, labels) (sort, PR / ROC / binned curves, AUROC, AP; its one synchronise included), between two
            CUDA events;
  * host:   the D2H copy of probs and labels, NumPy's argsort, the run ends and counts, the cut PR curve, the ROC curve, the
            binned curve by binary search, AUROC and AP, on a host clock that starts after a synchronise.
Reports the medians, the workspace ddfa_curve_workspace_bytes(n) and the peak device memory binary_curves allocates (workspace
plus outputs), checks that both paths give the same AUROC / AP (1e-12 relative), and prints one JSON line with the card's name,
power limit and maximum SM clock, read in the same run (and writes it to DIR/curve_cost.json)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepdfa_b200 import _lib  # noqa: E402
from deepdfa_b200.evaluator import binary_curves  # noqa: E402

SIZES = {"graph_split": 19_000, "node_split": 1_000_000, "arena": 10_400_000}
RATE = 0.06


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
    return {"device": q[0], "power_limit": q[1], "max_sm_clock": q[2]} if len(q) == 3 else {"device": torch.cuda.get_device_name(0)}


def host_curves(probs, labels, bins):
    """The host path: the same rules as binary_curves, in NumPy after a D2H copy."""
    p = probs.cpu().numpy()
    y = labels.cpu().numpy() == 1
    p = np.where(p == 0, np.float32(0), p)
    order = np.argsort(-p)
    ps, ys = p[order], y[order]
    ends = np.flatnonzero(np.append(ps[1:] != ps[:-1], True))
    tps = np.cumsum(ys, dtype=np.int64)[ends]
    fps = ends + 1 - tps
    thr = ps[ends]
    P, N = tps[-1], fps[-1]
    last = int(np.searchsorted(tps, P))
    sl = slice(0, last + 1)
    precision = np.append((tps / (tps + fps))[sl][::-1], 1.0)
    recall = np.append((tps / P)[sl][::-1], 0.0)
    fpr, tpr = np.append(0, fps) / N, np.append(0, tps) / P
    roc_thr = np.append(np.float32(thr[0] + np.float32(1)), thr)
    c = np.searchsorted(-thr, -bins, side="right")              # distinct thresholds >= t
    tp = np.where(c > 0, tps[c - 1], 0).astype(np.float64)
    fp = np.where(c > 0, fps[c - 1], 0).astype(np.float64)
    bp = np.append((tp + 1e-6) / (tp + fp + 1e-6), 1.0)
    br = np.append(tp / (P + 1e-6), 0.0)
    auroc = float(np.sum((fpr[1:] - fpr[:-1]) * (tpr[:-1] + tpr[1:]) / 2.0))
    ap = float(-np.sum((recall[1:] - recall[:-1]) * precision[:-1]))
    return (precision, recall, thr[sl][::-1]), (fpr, tpr, roc_thr), (bp, br), auroc, ap


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("curve_cost.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    info = card()
    bins = torch.linspace(0, 1.0, 100, dtype=torch.float32).numpy()
    rows = {}
    for name, n in SIZES.items():
        g = torch.Generator(device=dev).manual_seed(n)
        probs = torch.rand(n, device=dev, generator=g)
        labels = (torch.rand(n, device=dev, generator=g) < RATE).float()
        ws = _lib.lib().call("ddfa_curve_workspace_bytes", n)
        dev_res = binary_curves(probs, labels)                      # warm-up (module load, allocator)
        host_res = host_curves(probs, labels, bins)
        assert abs(dev_res["AUROC"] - host_res[3]) <= 1e-12 * abs(host_res[3]), (dev_res["AUROC"], host_res[3])
        assert abs(dev_res["AveragePrecision"] - host_res[4]) <= 1e-12 * abs(host_res[4])
        assert np.array_equal(dev_res["pr_curve"][2].cpu().numpy(), host_res[0][2])
        del dev_res
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t_dev, t_host = [], []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            r = binary_curves(probs, labels)
            b.record()
            torch.cuda.synchronize()
            t_dev.append(a.elapsed_time(b))
            del r
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_curves(probs, labels, bins)
            t_host.append((time.perf_counter() - t0) * 1e3)
        peak = torch.cuda.max_memory_allocated() - base
        rows[name] = {"n": n, "device_ms": float(np.median(t_dev)), "host_ms": float(np.median(t_host)),
                      "device_ms_all": [round(t, 3) for t in t_dev], "host_ms_all": [round(t, 3) for t in t_host],
                      "workspace_mib": ws / 2 ** 20, "peak_alloc_mib": peak / 2 ** 20}
        print(f"{name:12s} n={n:>9d}: device {rows[name]['device_ms']:8.3f} ms, host {rows[name]['host_ms']:9.3f} ms "
              f"({rows[name]['host_ms'] / rows[name]['device_ms']:.1f}x), workspace {ws / 2 ** 20:.1f} MiB, "
              f"peak {peak / 2 ** 20:.1f} MiB", flush=True)
        del probs, labels
    out = {**info, "positive_rate": RATE, "rounds": args.rounds, "sizes": rows}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "curve_cost.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
