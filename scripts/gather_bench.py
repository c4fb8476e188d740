"""GPU microbenchmark of the edge-gather launch-shape variants (ddfa_gather_sum_variant), forward (CSR) and
backward (transposed CSR, accumulate), L2-warm (the state inside a train step: h_t was just written) and
L2-cold (a 512 MB buffer is rewritten between launches).  Prints algorithmic GB/s per variant."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepdfa_b200 import synth
from deepdfa_b200._lib import lib
from deepdfa_b200.engine import _p, _stream_ptr, prepare_graph

DEV = "cuda:0"


def bench(fn, flush=None, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3)
    times.sort()
    return times[len(times) // 2], times[0]


def main():
    peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] \
        if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 3350.0
    L = lib()
    flush = torch.zeros(128 * 1024 * 1024, device=DEV)  # 512 MB > 50 MB L2
    for graphs, variable in ((256, False), (1024, False), (256, True)):
        g = synth.make_batch(graphs, 150, seed=1, variable=variable)
        dg = prepare_graph(g, DEV)
        N, E, D = g.num_nodes(), g.num_edges(), 128
        h = torch.randn(N, D, device=DEV)
        out = torch.empty(N, D, device=DEV)
        ref = torch.zeros(N, D, device=DEV).index_add_(0, g.edges()[1].to(DEV), h[g.edges()[0].to(DEV)])
        nbytes = E * D * 4 + N * D * 4 + E * 4 + (N + 1) * 4
        print(f"== graphs={graphs} variable={variable} N={N} E={E} bytes/launch={nbytes / 1e6:.2f} MB (peak {peaks:.0f} GB/s)")
        for v in (9, 3, 0, 10, 11):      # register path: default + two other launch shapes; 10 / 11: TMA-staged (gather_tma.cu)
            def fwd():
                L.call("ddfa_gather_sum_variant", v, _p(dg.indptr), _p(dg.indices), _p(h), N, D, _p(out), 0, _stream_ptr())
            def bwd():
                L.call("ddfa_gather_sum_variant", v, _p(dg.indptr_t), _p(dg.indices_t), _p(h), N, D, _p(out), 1, _stream_ptr())
            fwd(); torch.cuda.synchronize()
            err = float((out - ref).abs().max())
            wf, wfm = bench(fwd)
            cf, cfm = bench(fwd, flush)
            wb, _ = bench(bwd)
            print(f"  variant {v}: fwd warm {wf:6.1f} us ({nbytes / wf / 1e3:7.0f} GB/s, {nbytes / wf / 1e3 / peaks:4.2f} of peak) | "
                  f"fwd cold {cf:6.1f} us ({nbytes / cf / 1e3:7.0f} GB/s, {nbytes / cf / 1e3 / peaks:4.2f}) | bwd(acc) warm {wb:6.1f} us ({(nbytes + N * D * 4) / wb / 1e3:7.0f} GB/s) | err {err:.1e}")
        import ctypes
        bad = ctypes.c_int(0)
        L.call("ddfa_debug_read", 4, ctypes.addressof(bad), 4)
        print(f"  timed-out mbarrier waits in the TMA variants so far: {bad.value}")


if __name__ == "__main__":
    main()
