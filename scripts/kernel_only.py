"""Runs single tensor-core-engine kernels on a C0-sized batch, for `ncu -k regex:...` captures.
   python scripts/kernel_only.py fwd|bwd [graphs]
   DDFA_TRACE=1 additionally prints the in-kernel pipeline timeline (ddfa_debug_set key 2 / ddfa_debug_read)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepdfa_b200 import synth
from deepdfa_b200._lib import ENGINE_TCGEN05, lib
from deepdfa_b200.engine import _p, _stream_ptr, prepare_graph

DEV, D = "cuda:0", 128
# SM clock used to turn clock64() stamps into ns: the H100 SXM maximum unless DDFA_TRACE_GHZ gives the clock of the run
GHZ = float(os.environ.get("DDFA_TRACE_GHZ", "1.98"))
which = sys.argv[1] if len(sys.argv) > 1 else "fwd"
graphs = int(sys.argv[2]) if len(sys.argv) > 2 else 256
L = lib()
g = synth.make_batch(graphs, 150, seed=1)
dg = prepare_graph(g, DEV)
N = g.num_nodes()
torch.manual_seed(0)
k = 1.0 / D ** 0.5
wf = (torch.rand(3 * D, D, device=DEV) * 2 - 1) * k
whh = (torch.rand(3 * D, D, device=DEV) * 2 - 1) * k
bf, bih, bhh = [(torch.rand(3 * D, device=DEV) * 2 - 1) * k for _ in range(3)]
h = torch.tanh(torch.randn(N, D, device=DEV))
ib = L.call("ddfa_act_image_bytes", N)
s_img = torch.zeros(ib, dtype=torch.uint8, device=DEV); h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
o_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
out = torch.empty(N, D, device=DEV); gates = torch.rand(4, N, D, device=DEV)
st = _stream_ptr()
L.call("ddfa_act_to_image", _p(h), N, D, _p(h_img), st)
L.call("ddfa_gather_sum_image", _p(dg.indptr), _p(dg.indices), _p(h), N, D, _p(s_img), None, st)
if which == "fwd":
    wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D, ENGINE_TCGEN05)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare", _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), D, ENGINE_TCGEN05, _p(ws), wsb, st)
    gpk = torch.zeros(L.call("ddfa_gru_gates_packed_bytes", N, D), dtype=torch.uint8, device=DEV)

    def fwd_v2(train):      # the form the training / inference drivers use: h from the image, image out, packed gates when training
        L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D, None, _p(o_img), _p(gpk) if train else None,
               _p(ws), wsb, st)
    for i in range(6):
        fwd_v2(i % 2 == 1)
else:
    wsb = L.call("ddfa_gru_step_bwd_workspace_bytes", N, D, ENGINE_TCGEN05)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare_bwd", _p(wf), _p(whh), D, ENGINE_TCGEN05, _p(ws), wsb, st)
    dh_o = torch.randn(N, D, device=DEV); ds = torch.empty(N, D, device=DEV); dh = torch.empty(N, D, device=DEV)
    ds_p = torch.randn(N, D, device=DEV)     # the previous step's ds: its transposed gather is folded into the call
    acc = [torch.zeros(3 * D, D, device=DEV), torch.zeros(3 * D, device=DEV), torch.zeros(3 * D, device=DEV),
           torch.zeros(3 * D, D, device=DEV), torch.zeros(3 * D, device=DEV)]
    for i in range(4):
        L.call("ddfa_gru_step_bwd_image", _p(dh_o), _p(ds_p), _p(dg.indptr_t), _p(dg.indices_t), _p(h), _p(h_img), _p(s_img), _p(gates), _p(dg.indptr),
               N, D, _p(ds), _p(dh), _p(acc[0]), _p(acc[1]), _p(acc[2]), _p(acc[3]), _p(acc[4]), _p(ws), wsb, 1 if i == 0 else 2, st)
torch.cuda.synchronize()
print("done", which, N)


def dump_trace(key, label):
    import numpy as np
    CT, TL, EV = 132, 12, 16
    buf = np.zeros(CT * TL * EV, dtype=np.int64)
    L.call("ddfa_debug_read", key, buf.ctypes.data, buf.nbytes)
    t = buf.reshape(CT, TL, EV).astype(np.float64)
    ghz = GHZ
    names = ["start", "prod:first copy issued", "prod:last copy issued", "mma:acc buffer free", "mma:first operand landed",
             "mma:last operand landed", "mma:tile committed", "epi:iteration begin", "epi:accumulator ready", "epi:stages released",
             "epi:iteration end"]
    print(f"---- {label}: per-tile timeline, ns since the CTA's kernel start (SM clock / {ghz} GHz)")
    for cta in (0, 1, 5, 66, 131):
        t0 = t[cta, 0, 0]
        print(f"CTA {cta}:")
        for k in range(TL):
            if t[cta, k, 6] == 0:
                break
            print("   tile %2d " % k + " ".join("%7.0f" % ((t[cta, k, e] - t0) / ghz) for e in range(1, 11)))
    # averages over CTAs, for steady-state tiles 2..6
    def span(a, b, k0=2, k1=7):
        d = (t[:, k0:k1, b] - t[:, k0:k1, a]) / ghz
        ok = (t[:, k0:k1, 6] != 0)
        return d[ok].mean(), np.percentile(d[ok], 90)
    print("events: " + " | ".join(f"{i + 1}={n}" for i, n in enumerate(names[1:])))
    for a, b, what in ((1, 4, "first copy issue -> landed"), (1, 2, "producer: first -> last copy issued"), (4, 5, "mma: first -> last operand landed"),
                       (5, 6, "mma: last operand -> commit issued"), (6, 8, "commit issued -> epilogue sees accumulator"),
                       (8, 9, "epilogue: stage release"), (9, 10, "epilogue: after drain -> iteration end"), (7, 10, "epilogue iteration"),
                       (7, 8, "epilogue: begin -> accumulator ready (prefetch + wait)")):
        m, p90 = span(a, b)
        print(f"   {what:56s} mean {m:8.0f} ns   p90 {p90:8.0f} ns")
    per_tile = (t[:, 1:7, 10] - t[:, 0:6, 10]) / ghz
    ok = (t[:, 1:7, 6] != 0)
    print(f"   epilogue end-to-end period per tile: mean {per_tile[ok].mean():.0f} ns; kernel span (CTA 0): {(t[0, :, 10].max() - t[0, 0, 0]) / ghz:.0f} ns")


if os.environ.get("DDFA_TRACE"):
    L.call("ddfa_debug_set", 2, 1)
    if which == "fwd":
        for train in (False, True):
            fwd_v2(train)
            torch.cuda.synchronize()
            dump_trace(3, "gru_fwd3_kernel " + ("train" if train else "infer"))
    else:
        L.call("ddfa_gru_step_bwd_image", _p(dh_o), _p(ds_p), _p(dg.indptr_t), _p(dg.indices_t), _p(h), _p(h_img), _p(s_img), _p(gates), _p(dg.indptr),
               N, D, _p(ds), _p(dh), _p(acc[0]), _p(acc[1]), _p(acc[2]), _p(acc[3]), _p(acc[4]), _p(ws), wsb, 2, st)
        torch.cuda.synchronize()
        dump_trace(2, "dgrad_kernel")
        L.call("ddfa_debug_set", 2, 2)
        L.call("ddfa_gru_step_bwd_image", _p(dh_o), _p(ds_p), _p(dg.indptr_t), _p(dg.indices_t), _p(h), _p(h_img), _p(s_img), _p(gates), _p(dg.indptr),
               N, D, _p(ds), _p(dh), _p(acc[0]), _p(acc[1]), _p(acc[2]), _p(acc[3]), _p(acc[4]), _p(ws), wsb, 2, st)
        torch.cuda.synchronize()
        import numpy as np
        buf = np.zeros(132 * 12 * 16, dtype=np.int64)
        L.call("ddfa_debug_read", 2, buf.ctypes.data, buf.nbytes)
        t = buf.reshape(132, 12, 16).astype(np.float64) / GHZ
        print("---- wgrad_kernel (gate block 0 of dW'): ns since kernel start: B issue | A issue | B landed | A landed | A landed | tile MMAs issued")
        for cta in (0, 1, 11, 21):
            t0 = t[cta, 0, 0]
            print(f"CTA {cta}: epilogue begins {t[cta, 0, 8] - t0:.0f}, ends {t[cta, 0, 10] - t0:.0f}")
            for k in range(12):
                if t[cta, k, 6] == 0:
                    break
                print("   tile %2d " % k + " ".join("%7.0f" % (t[cta, k, e] - t0) for e in (1, 2, 3, 4, 5, 6)))
    L.call("ddfa_debug_set", 2, 0)
