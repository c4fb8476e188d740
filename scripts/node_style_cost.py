"""Cost of a label_style="node" training step at the benchmark's C1 batch, with CUDA events.

    python scripts/node_style_cost.py [--rounds 5] [--steps 20]

For ``undersample_node_on_loss_factor`` None and 1.0, two arms on the same C1 batch (1024 graphs x 150 nodes, D = 128, T = 8,
L = 2, tensor-core engine), timed in alternating rounds of ``--steps`` steps each:
  * fused:  FusedTrainer(use_cuda_graph=True) replaying its captured step (the loss rows drawn on the device);
  * module: module.training_step + loss.backward() + torch.optim.Adam (the rows drawn on the host by random.sample).
Also times the fused trainer's head forward (ddfa_node_head_fwd) and backward (ddfa_node_head_bwd) alone on the step's own
buffers.  Prints one JSON line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import engine as E  # noqa: E402
from deepdfa_b200 import synth  # noqa: E402

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


def module(factor, dev):
    torch.manual_seed(0)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, label_style="node", concat_all_absdf=True, positive_weight=2.0,
                               undersample_node_on_loss_factor=factor, engine="tcgen05").to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("node_style_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    batch = synth.make_batch(1024, 150, seed=0).to(dev)
    med = lambda xs: sorted(xs)[len(xs) // 2]                   # noqa: E731
    result = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "nodes": batch.num_nodes(),
              "vulnerable_nodes": int(batch.ndata["_VULN"].sum())}
    for factor in (None, 1.0):
        m_f = module(factor, dev)
        tr = D.FusedTrainer(m_f, use_cuda_graph=True)
        for _ in range(3):                                      # eager warm-up, capture, replay
            tr.step(batch)
        rows = int(tr.last_loss_rows().numel())
        m_m = module(factor, dev)
        opt = torch.optim.Adam(m_m.parameters(), lr=1e-3, weight_decay=1e-2)
        random.seed(0)

        def module_step():
            opt.zero_grad()
            loss = m_m.training_step((batch, {}), 0)
            loss.backward()
            opt.step()
        module_step()
        t_fused, t_module = [], []
        for _ in range(args.rounds):
            t_fused.append(timed(lambda: tr.step(batch), args.steps))
            t_module.append(timed(module_step, args.steps))
        # the head alone, on the trainer's own buffers (the last step's rows and activations)
        ws, N, Dm = tr.ws, batch.num_nodes(), m_f._D
        x, h_T = ws.get("x", (N, Dm)), ws.get("h_final", (N, Dm))
        rows_buf = ws.get("node_rows", (N,), torch.int32)
        logits, act = E.node_head_fwd(tr.params, x, h_T, rows_buf, tr._num_rows, alloc=ws)
        dl = ws.get("node_dlogits", (N,))
        head_fwd = timed(lambda: E.node_head_fwd(tr.params, x, h_T, rows_buf, tr._num_rows, alloc=ws), 50)
        head_bwd = timed(lambda: E.node_head_bwd(tr.params, tr.grads, dl, x, h_T, rows_buf, tr._num_rows, act,
                                                 alloc=ws), 50)
        key = "none" if factor is None else f"{factor:g}"
        result[f"factor_{key}"] = {"loss_rows": rows, "fused_ms": [round(v, 3) for v in t_fused], "module_ms": [round(v, 3) for v in t_module],
                                   "fused_median_ms": round(med(t_fused), 3), "module_median_ms": round(med(t_module), 3),
                                   "head_fwd_ms": round(head_fwd, 3), "head_bwd_ms": round(head_bwd, 3),
                                   "head_share_of_fused_step": round((head_fwd + head_bwd) / med(t_fused), 4)}
        del tr, m_f, m_m, opt
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
