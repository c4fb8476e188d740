"""GPU diagnostic for the tensor-core GRU-step kernel: structured inputs that expose descriptor / swizzle /
fragment-layout mistakes (gh_n is a raw accumulator + bias, so with Whh_n = I it must reproduce h exactly),
then a random case against the fp64 formula.  Run under `timeout`; prints a compact error map."""
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepdfa_b200._lib import ENGINE_SIMT, ENGINE_TCGEN05, lib
from deepdfa_b200.engine import _p, _stream_ptr

DEV = "cuda:0"
D = 128


def run_step(engine, s, h, indptr, wf, bf, bih, whh, bhh):
    L = lib()
    N = s.shape[0]
    wsb = max(L.call("ddfa_gru_step_workspace_bytes", N, D, engine), 16)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare", _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), D, engine, _p(ws), wsb, _stream_ptr())
    h_out = torch.full((N, D), float("nan"), device=DEV)
    gates = torch.full((4, N, D), float("nan"), device=DEV)
    L.call("ddfa_gru_step_fwd", _p(s), _p(h), _p(indptr), _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), N, D, _p(h_out), _p(gates),
           _p(ws), wsb, engine, _stream_ptr())
    torch.cuda.synchronize()
    return h_out, gates


def errmap(name, got, ref, rb=32, cb=32):
    err = (got.double() - ref.double()).abs()
    err = torch.nan_to_num(err, nan=1e9)
    print(f"{name}: max err {float(err.max()):.3e}  (ref max {float(ref.abs().max()):.3e}), nan count {int(torch.isnan(got).sum())}")
    if float(err.max()) > 1e-4:
        n = (got.shape[0] // rb) * rb
        blocks = err[:n].reshape(n // rb, rb, D // cb, cb).amax(dim=(1, 3))
        print("  block max-error map (rows x cols, blocks of %dx%d):" % (rb, cb))
        for r in range(min(blocks.shape[0], 8)):
            print("   ", " ".join(f"{float(v):9.2e}" for v in blocks[r]))


def main():
    torch.manual_seed(0)
    N = 300   # 2 full tiles + a ragged one
    indptr = torch.arange(N + 1, dtype=torch.int32, device=DEV) * 2     # indeg = 2 everywhere
    z3 = torch.zeros(3 * D, device=DEV)
    # --- test 1: Whh_n = I, everything else zero: gh_n must equal h; gin = 0, r = z = 0.5
    h = (torch.arange(N * D, device=DEV, dtype=torch.float32).reshape(N, D) % 977) / 977.0 - 0.5
    s = torch.zeros(N, D, device=DEV)
    whh = torch.zeros(3 * D, D, device=DEV); whh[2 * D:] = torch.eye(D, device=DEV)
    wf = torch.zeros(3 * D, D, device=DEV)
    _, g = run_step(ENGINE_TCGEN05, s, h, indptr, wf, z3, z3, whh, z3)
    errmap("T1 gh_n == h (Whh_n = I)", g[3], h)
    errmap("T1 r == 0.5", g[0], torch.full_like(h, 0.5))
    # --- test 2: W'_n = I with s pattern: gin -> n = tanh(gin); check atanh(n) == s
    s2 = ((torch.arange(N * D, device=DEV, dtype=torch.float32).reshape(N, D) * 7) % 1013) / 1013.0 - 0.5
    wf2 = torch.zeros(3 * D, D, device=DEV); wf2[2 * D:] = torch.eye(D, device=DEV)
    _, g = run_step(ENGINE_TCGEN05, s2, torch.zeros(N, D, device=DEV), indptr, wf2, z3, z3, torch.zeros(3 * D, D, device=DEV), z3)
    errmap("T2 atanh(n) == s (W'_n = I)", torch.atanh(g[2].clamp(-0.999999, 0.999999)), s2)
    # --- test 3: W'_r = I and Whh_r = 2I: logit(r) == s + 2h
    wf3 = torch.zeros(3 * D, D, device=DEV); wf3[:D] = torch.eye(D, device=DEV)
    whh3 = torch.zeros(3 * D, D, device=DEV); whh3[:D] = 2 * torch.eye(D, device=DEV)
    _, g = run_step(ENGINE_TCGEN05, s2, h, indptr, wf3, z3, z3, whh3, z3)
    errmap("T3 logit(r) == s + 2h", torch.logit(g[0].clamp(1e-6, 1 - 1e-6)), s2 + 2 * h)
    # --- test 4: random, vs SIMT engine and fp64
    k = 1.0 / D ** 0.5
    wf4 = (torch.rand(3 * D, D, device=DEV) * 2 - 1) * k * 1.5
    whh4 = (torch.rand(3 * D, D, device=DEV) * 2 - 1) * k
    bf4, bih4, bhh4 = [(torch.rand(3 * D, device=DEV) * 2 - 1) * k for _ in range(3)]
    s4 = torch.randn(N, D, device=DEV) * 2
    h4 = torch.tanh(torch.randn(N, D, device=DEV))
    ho_tc, g_tc = run_step(ENGINE_TCGEN05, s4, h4, indptr, wf4, bf4, bih4, whh4, bhh4)
    ho_si, g_si = run_step(ENGINE_SIMT, s4, h4, indptr, wf4, bf4, bih4, whh4, bhh4)
    sd, hd = s4.double(), h4.double()
    gi = sd @ wf4.double().t() + 2.0 * bf4.double() + bih4.double()
    gh = hd @ whh4.double().t() + bhh4.double()
    r = torch.sigmoid(gi[:, :D] + gh[:, :D]); zz = torch.sigmoid(gi[:, D:2 * D] + gh[:, D:2 * D])
    nn = torch.tanh(gi[:, 2 * D:] + r * gh[:, 2 * D:])
    ref = (1 - zz) * nn + zz * hd
    errmap("T4 h_out tcgen05 vs fp64", ho_tc, ref)
    errmap("T4 h_out simt    vs fp64", ho_si, ref)
    errmap("T4 gh_n  tcgen05 vs fp64", g_tc[3], gh[:, 2 * D:])
    errmap("T4 gh_n  simt    vs fp64", g_si[3], gh[:, 2 * D:])
    # --- test 5: backward, tcgen05 vs SIMT engine (the SIMT backward is pinned against fp64 autograd in tests/)
    def run_bwd(engine, N_, dh_o, h_, s_, gates_, ip_):
        L = lib()
        wsb = max(L.call("ddfa_gru_step_bwd_workspace_bytes", N_, D, engine), 16)
        ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare_bwd", _p(wf4), _p(whh4), D, engine, _p(ws), wsb, _stream_ptr())
        outs = {"ds": torch.full((N_, D), float("nan"), device=DEV), "dh": torch.full((N_, D), float("nan"), device=DEV),
                "dwf": torch.zeros(3 * D, D, device=DEV), "dbf": torch.zeros(3 * D, device=DEV), "dbih": torch.zeros(3 * D, device=DEV),
                "dwhh": torch.zeros(3 * D, D, device=DEV), "dbhh": torch.zeros(3 * D, device=DEV)}
        def call():
            L.call("ddfa_gru_step_bwd", _p(dh_o), _p(h_), _p(s_), _p(gates_), _p(ip_), _p(wf4), _p(whh4), N_, D, _p(outs["ds"]), _p(outs["dh"]),
                   _p(outs["dwf"]), _p(outs["dbf"]), _p(outs["dbih"]), _p(outs["dwhh"]), _p(outs["dbhh"]), _p(ws), wsb, engine, _stream_ptr())
        call()
        torch.cuda.synchronize()
        return outs, call
    dh_o = torch.randn(N, D, device=DEV)
    o_tc, _ = run_bwd(ENGINE_TCGEN05, N, dh_o, h4, s4, g_si, indptr)
    o_si, _ = run_bwd(ENGINE_SIMT, N, dh_o, h4, s4, g_si, indptr)
    for k in o_tc:
        if o_tc[k].dim() == 2 and o_tc[k].shape[0] == N:
            errmap(f"T5 bwd {k} tcgen05 vs simt", o_tc[k], o_si[k])
        else:
            e = float((o_tc[k].double() - o_si[k].double()).abs().max()); sc = float(o_si[k].abs().max())
            print(f"T5 bwd {k}: max err {e:.3e} (ref max {sc:.3e}), nan {int(torch.isnan(o_tc[k]).sum())}")
            if o_tc[k].dim() == 2 and e > 1e-3 * max(sc, 1):
                err = (o_tc[k] - o_si[k]).abs().reshape(3, 4, 32, 4, 32).amax(dim=(2, 4))
                print("   block map [gate][row32][col32]:", [[f"{float(x):.1e}" for x in r_.flatten()] for r_ in err])
    # timing
    N2 = 38400
    s5 = torch.randn(N2, D, device=DEV); h5 = torch.tanh(torch.randn(N2, D, device=DEV)); d5 = torch.randn(N2, D, device=DEV)
    g5 = torch.rand(4, N2, D, device=DEV)
    ip5 = torch.arange(N2 + 1, dtype=torch.int32, device=DEV) * 2
    for eng, name in ((ENGINE_TCGEN05, "tcgen05"), (ENGINE_SIMT, "simt")):
        _, call = run_bwd(eng, N2, d5, h5, s5, g5, ip5)
        for _ in range(3):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            call()
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / 10 * 1e3
        print(f"timing bwd {name} N={N2}: {us:.1f} us/step ({2 * 2.0 * N2 * 6 * D * D / us / 1e6:.1f} TFLOP/s algorithmic)")
    # image-path kernels alone (what the training driver calls)
    def timeit(fn, iters=20):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e3
    from deepdfa_b200 import synth
    from deepdfa_b200.engine import prepare_graph
    for graphs in (256, 1024):
        gb = synth.make_batch(graphs, 150, seed=1)
        dgb = prepare_graph(gb, DEV)
        Nb = gb.num_nodes()
        L = lib()
        hb = torch.tanh(torch.randn(Nb, D, device=DEV)); ob = torch.empty(Nb, D, device=DEV); gt = torch.empty(4, Nb, D, device=DEV)
        ib = L.call("ddfa_act_image_bytes", Nb)
        s_img = torch.zeros(ib, dtype=torch.uint8, device=DEV); h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        o_img = torch.zeros(ib, dtype=torch.uint8, device=DEV); s_f = torch.empty(Nb, D, device=DEV)
        wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D, ENGINE_TCGEN05)
        ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare", _p(wf4), _p(bf4), _p(bih4), _p(whh4), _p(bhh4), D, ENGINE_TCGEN05, _p(ws), wsb, _stream_ptr())
        L.call("ddfa_act_to_image", _p(hb), Nb, D, _p(h_img), _stream_ptr())
        t_g = timeit(lambda: L.call("ddfa_gather_sum", _p(dgb.indptr), _p(dgb.indices), _p(hb), Nb, D, _p(s_f), 0, _stream_ptr()))
        t_gi = timeit(lambda: L.call("ddfa_gather_sum_image", _p(dgb.indptr), _p(dgb.indices), _p(hb), Nb, D, _p(s_img), None, _stream_ptr()))
        t_gif = timeit(lambda: L.call("ddfa_gather_sum_image", _p(dgb.indptr), _p(dgb.indices), _p(hb), Nb, D, _p(s_img), _p(s_f), _stream_ptr()))
        # check the image against the fp32 gather through the fp32-input reference path
        t_ti = timeit(lambda: L.call("ddfa_act_to_image", _p(hb), Nb, D, _p(h_img), _stream_ptr()))
        t_f0 = timeit(lambda: L.call("ddfa_gru_step_fwd_image", _p(s_img), _p(h_img), _p(hb), _p(dgb.indptr), Nb, D, _p(ob), None, None, _p(ws), wsb, _stream_ptr()))
        t_f1 = timeit(lambda: L.call("ddfa_gru_step_fwd_image", _p(s_img), _p(h_img), _p(hb), _p(dgb.indptr), Nb, D, _p(ob), _p(o_img), _p(gt), _p(ws), wsb, _stream_ptr()))
        fl = 2.0 * Nb * 6 * D * D
        print(f"image path N={Nb}: gather fp32 {t_g:.1f} us | gather->image {t_gi:.1f} us | gather->image+fp32 {t_gif:.1f} us | to_image {t_ti:.1f} us | "
              f"gru_fwd_image infer {t_f0:.1f} us ({fl / t_f0 / 1e6:.0f} TFLOP/s alg) | train(+img+gates) {t_f1:.1f} us ({fl / t_f1 / 1e6:.0f} TFLOP/s alg)")
        # correctness of the image chain vs the fp32-in entry point
        ref_out = torch.empty(Nb, D, device=DEV)
        wsb2 = L.call("ddfa_gru_step_workspace_bytes", Nb, D, ENGINE_TCGEN05); ws2 = torch.zeros(wsb2, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare", _p(wf4), _p(bf4), _p(bih4), _p(whh4), _p(bhh4), D, ENGINE_TCGEN05, _p(ws2), wsb2, _stream_ptr())
        L.call("ddfa_gru_step_fwd", _p(s_f), _p(hb), _p(dgb.indptr), _p(wf4), _p(bf4), _p(bih4), _p(whh4), _p(bhh4), Nb, D, _p(ref_out), None, _p(ws2), wsb2, ENGINE_TCGEN05, _stream_ptr())
        torch.cuda.synchronize()
        print(f"   image chain vs fp32-in entry: max diff {float((ob - ref_out).abs().max()):.3e}")
    for eng, name in ((ENGINE_TCGEN05, "tcgen05"), (ENGINE_SIMT, "simt")):
        N2 = 38400
        s5 = torch.randn(N2, D, device=DEV); h5 = torch.tanh(torch.randn(N2, D, device=DEV))
        ip = torch.arange(N2 + 1, dtype=torch.int32, device=DEV) * 2
        L = lib()
        wsb = max(L.call("ddfa_gru_step_workspace_bytes", N2, D, eng), 16)
        ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare", _p(wf4), _p(bf4), _p(bih4), _p(whh4), _p(bhh4), D, eng, _p(ws), wsb, _stream_ptr())
        out = torch.empty(N2, D, device=DEV); gt = torch.empty(4, N2, D, device=DEV)
        for gates in (None, gt):
            for _ in range(3):
                L.call("ddfa_gru_step_fwd", _p(s5), _p(h5), _p(ip), _p(wf4), _p(bf4), _p(bih4), _p(whh4), _p(bhh4), N2, D, _p(out), _p(gates),
                       _p(ws), wsb, eng, _stream_ptr())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                L.call("ddfa_gru_step_fwd", _p(s5), _p(h5), _p(ip), _p(wf4), _p(bf4), _p(bih4), _p(whh4), _p(bhh4), N2, D, _p(out), _p(gates),
                       _p(ws), wsb, eng, _stream_ptr())
            e1.record(); torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 20 * 1e3
            fl = 2.0 * N2 * 6 * D * D
            print(f"timing {name} N={N2} gates={'yes' if gates is not None else 'no'}: {us:.1f} us/step  ({fl / us / 1e6:.1f} TFLOP/s algorithmic)")


if __name__ == "__main__":
    main()
