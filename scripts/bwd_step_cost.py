"""Cost of the fused backward GRU step (bwd_step_fused_kernel) at the benchmark's C1 batch, in the engine's default mode.

    python scripts/bwd_step_cost.py [--calls 20] [--replays 10]
    DDFA_LIB_PATH=<other build>/libddfa_b200.so python scripts/bwd_step_cost.py      # A/B of two builds, alternately in one session

Calls ddfa_gru_step_bwd_image_v2 on the packed saved state (h as the activation image, the previous step's ds folded in, the
q images kept for the batched weight-gradient launch, so the call is the fused kernel alone), as the training driver does at
steps t > 0.  Prints one JSON line: the card, its power limit and maximum SM clock, and the mean time per call from CUDA events
around replays of a CUDA graph of --calls calls.  With DDFA_TRACE=1 it also prints the per-tile phase breakdown of one eager
call from the kernel's SM-clock stamps (ddfa_debug_set(2, 1)), averaged over every CTA's steady-state tiles 2-6:
  start -> handover      phase A (gate backward and the folded gather) and the cluster barrier (event 11)
  handover -> first q    waiting for the first q tile of phase B (event 4)
  first q -> last MMAs   the dgrad MMAs (events 6 / 8)
  accumulator -> end     the ds / dh epilogue (event 9 -> event 10)
  period                 iteration end to iteration end
and where phase A and the epilogue's copy issue end:
  start -> last phase A  the CTA's last warp has read its phase-A rows (event 14, an atomic max over the warps)
  last phase A -> handover   the cluster barrier: the other CTAs' phase A and the q / dh' * z stores made visible
  accumulator -> issued (wg 0 / wg 1)   warpgroup 0 / 1 has issued its ds / dh copies (events 12 / 13)"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepdfa_b200 import synth  # noqa: E402
from deepdfa_b200._lib import ENGINE_TCGEN05, lib  # noqa: E402
from deepdfa_b200.engine import _p, prepare_graph  # noqa: E402

DEV, D = "cuda:0", 128
KEEP0 = 16                     # DDFA_WGRAD_KEEP(0): keep the q images, no weight-gradient launch inside the call
CT, TL, EV = 132, 12, 16       # the trace buffer: [CTA][tile][event] (tc_common.cuh)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"device": q[0], "power_limit": q[1], "max_sm_clock": q[2]}


def phases(t):
    """Per-tile spans in SM cycles over tiles 2-6 of every CTA that ran them."""
    k = np.arange(2, 7)
    ok = (t[:, k, 10] != 0) & (t[:, k - 1, 10] != 0)
    spans = {"start_to_handover": t[:, k, 11] - t[:, k - 1, 10], "handover_to_first_q": t[:, k, 4] - t[:, k, 11],
             "first_q_to_last_mmas": t[:, k, 6] - t[:, k, 4], "accumulator_to_end": t[:, k, 10] - t[:, k, 9],
             "period": t[:, k, 10] - t[:, k - 1, 10],
             "start_to_last_phase_a": t[:, k, 14] - t[:, k - 1, 10], "last_phase_a_to_handover": t[:, k, 11] - t[:, k, 14],
             "accumulator_to_issued_wg0": t[:, k, 12] - t[:, k, 9], "accumulator_to_issued_wg1": t[:, k, 13] - t[:, k, 9]}
    return {n: round(float(v[ok].mean()), 0) for n, v in spans.items()}, int(ok.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20, help="calls captured in the CUDA graph")
    ap.add_argument("--replays", type=int, default=10, help="timed replays of the graph (calls x replays >= 200)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bwd_step_cost.py measures on the GPU; no CUDA device found")
    L = lib()
    g = synth.make_batch(1024, 150, 2.0, 1002, seed=0)            # the benchmark's C1 batch
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    gen = torch.Generator().manual_seed(0)
    k = 1.0 / D ** 0.5
    mk = lambda *sh: ((torch.rand(*sh, generator=gen) * 2 - 1) * k).to(DEV)
    wf, bf, bih, whh, bhh = mk(3 * D, D), mk(3 * D), mk(3 * D), mk(3 * D, D), mk(3 * D)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        st = side.cuda_stream
        ib = L.call("ddfa_act_image_bytes", N)
        h32 = torch.tanh(torch.randn(N, D, generator=gen)).to(DEV)
        h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        L.call("ddfa_act_to_image", _p(h32), N, D, _p(h_img), st)
        s_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gather_sum_image_src", _p(dg.indptr), _p(dg.indices), _p(h_img), N, D, _p(s_img), st)
        wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D, ENGINE_TCGEN05)
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare", _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), D, ENGINE_TCGEN05, _p(ws), wsb, st)
        gates = torch.empty(L.call("ddfa_gru_gates_packed_bytes", N, D), dtype=torch.uint8, device=DEV)
        o_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D, None, _p(o_img), _p(gates), _p(ws), wsb, st)
        wsb_b = L.call("ddfa_gru_step_bwd_workspace_bytes", N, D, ENGINE_TCGEN05)
        ws_b = torch.empty(wsb_b, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare_bwd", _p(wf), _p(whh), D, ENGINE_TCGEN05, _p(ws_b), wsb_b, st)
        dpart, ds_prev = torch.randn(N, D, generator=gen).to(DEV), torch.randn(N, D, generator=gen).to(DEV)
        ds, dh = torch.empty(N, D, device=DEV), torch.empty(N, D, device=DEV)
        grads = [torch.zeros(3 * D, D, device=DEV), torch.zeros(3 * D, device=DEV), torch.zeros(3 * D, device=DEV),
                 torch.zeros(3 * D, D, device=DEV), torch.zeros(3 * D, device=DEV)]

        def call():
            L.call("ddfa_gru_step_bwd_image_v2", _p(dpart), _p(ds_prev), _p(dg.indptr_t), _p(dg.indices_t), None, _p(h_img), _p(s_img),
                   _p(gates), _p(dg.indptr), N, D, _p(ds), _p(dh), *[_p(x) for x in grads], _p(ws_b), wsb_b, KEEP0, st)

        for _ in range(3):
            call()
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            for _ in range(args.calls):
                call()
        graph.replay()
        side.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(side)
        for _ in range(args.replays):
            graph.replay()
        b.record(side)
        side.synchronize()
        res = {**card(), "lib": str(L.path), "nodes": N, "tiles": (N + 127) // 128,
               "calls": args.calls * args.replays, "us_per_call": round(a.elapsed_time(b) * 1e3 / (args.calls * args.replays), 1)}
        if os.environ.get("DDFA_TRACE"):
            L.call("ddfa_debug_set", 2, 1)
            try:
                call()
                side.synchronize()
                buf = np.zeros(CT * TL * EV, dtype=np.int64)
                L.call("ddfa_debug_read", 2, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes)
            finally:
                L.call("ddfa_debug_set", 2, 0)
            res["tile_cycles"], res["tiles_averaged"] = phases(buf.reshape(CT, TL, EV).astype(np.float64))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
