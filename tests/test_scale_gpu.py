"""GPU: the kernels at training-batch sizes and hub degrees, against fp64 host references of the same operations.

The other GPU tests run the persistent tensor-core kernels at sizes where their loops barely turn.  Here every kernel runs at
the trip counts of the benchmark's C1 batch (about 157 000 nodes: 37-38 gate-backward blocks and forward / dgrad tiles per CTA,
hundreds of weight-gradient tiles per CTA) and just past the gate backward's ring-refill threshold, on batches with hub rows
that take every long-neighbour-list path of the edge gathers (tests/scale_batches.py; tests/test_scale_premises.py checks on
the CPU that the shapes still reach these counts).  Every test prints its worst error against its bound."""
import ctypes

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import synth
from deepdfa_b200._lib import (ENGINE_SIMT, ENGINE_TCGEN05, TUNE_GATE_BWD_TMA, TUNE_GATHER_SRC_GROUPS, TUNE_GATHER_VARIANT, DdfaError,
                               lib)
from deepdfa_b200.engine import _p, _stream_ptr, prepare_graph
from oracle import ggnn_oracle as O
from scale_batches import MODULE_C1, hub_batch
from tc_images import decode_gates, decode_image

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
U = 2.0 ** -24                 # unit roundoff of fp32
NUM_VARIANTS = 12              # ddfa_gather_sum_variant: 0-9 register path, 10-11 TMA-staged


def _gather_refs(h, src, dst, N):
    """fp64 sum over in-edges, the sum of the magnitudes and the in-degree — the ingredients of the summation error bound."""
    h64 = h.double()
    ref = torch.zeros(N, h.shape[1], dtype=torch.float64).index_add_(0, dst, h64[src])
    mag = torch.zeros(N, h.shape[1], dtype=torch.float64).index_add_(0, dst, h64.abs()[src])
    return ref, mag, torch.bincount(dst, minlength=N).double()[:, None]


def _ratio(err, bound):
    """Largest err / bound (0 where both are 0, inf where only the bound is)."""
    return float(torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0)).max())


def _orientations(g, dg):
    src, dst = g.edges()
    return (("csr", dg.indptr, dg.indices, src, dst), ("transposed", dg.indptr_t, dg.indices_t, dst, src))


# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["threshold", "c1"])
def test_gather_variants_at_hub_degrees(shape):
    """All twelve launch variants of the width-128 edge gather, plain and accumulating, over the CSR and the transposed CSR of a
    hub batch.  Each sums its row's neighbours in neighbour order, so all twelve give the same bits; the sum is held to the
    a-priori bound of recursive fp32 summation, |err| <= 2 (deg + acc) u (sum |h_src| + acc |out_0|)."""
    g = hub_batch(shape)
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    gen = torch.Generator().manual_seed(N)
    h, base = torch.randn(N, 128, generator=gen), torch.randn(N, 128, generator=gen)
    hd, based = h.to(DEV), base.to(DEV)
    L, st = lib(), _stream_ptr()
    default = L.call("ddfa_tuning_get", TUNE_GATHER_VARIANT)
    worst = {}
    for orient, ip, ix, s_, d_ in _orientations(g, dg):
        ref, mag, deg = _gather_refs(h, s_, d_, N)
        for acc in (0, 1):
            def fresh():
                return based.clone() if acc else torch.full((N, 128), float("nan"), device=DEV)
            outs = []
            for v in range(NUM_VARIANTS):
                out = fresh()
                L.call("ddfa_gather_sum_variant", v, _p(ip), _p(ix), _p(hd), N, 128, _p(out), acc, st)
                outs.append(out)
            for v in range(1, NUM_VARIANTS):
                assert torch.equal(outs[v], outs[0]), (orient, acc, v)
            r = ref + base.double() if acc else ref
            bound = 2 * (deg + acc) * U * (mag + base.double().abs() if acc else mag)
            worst[f"{orient},acc={acc}"] = _ratio((outs[0].cpu().double() - r).abs(), bound)
            # the production entry point runs whichever variant the tuning key selects
            try:
                for v in range(NUM_VARIANTS):
                    L.call("ddfa_tuning_set", TUNE_GATHER_VARIANT, v)
                    out = fresh()
                    L.call("ddfa_gather_sum", _p(ip), _p(ix), _p(hd), N, 128, _p(out), acc, st)
                    assert torch.equal(out, outs[v]), (orient, acc, v)
            finally:
                L.call("ddfa_tuning_set", TUNE_GATHER_VARIANT, default)
            del outs
    torch.cuda.synchronize()
    timed_out = ctypes.c_int(-1)
    L.call("ddfa_debug_read", 4, ctypes.addressof(timed_out), ctypes.sizeof(timed_out))
    print(f"gather variants, {shape} N={N}: worst |err| / bound: " + ", ".join(f"{k}={v:.2f}" for k, v in worst.items()))
    assert timed_out.value == 0                 # no bounded mbarrier wait of the TMA variants ran out
    assert max(worst.values()) <= 1.0, worst
    with pytest.raises(DdfaError, match="unknown variant 12"):
        L.call("ddfa_gather_sum_variant", NUM_VARIANTS, _p(dg.indptr), _p(dg.indices), _p(hd), N, 128, _p(based), 0, st)


@pytest.mark.parametrize("shape", ["threshold", "c1"])
def test_image_gathers_at_hub_degrees(shape):
    """The gathers that write activation images (fp32 rows in; image in, with 1, 2 and 4 row groups per warp) on a hub batch,
    both orientations.  The images start as garbage: every byte, the zero rows past N included, must be written."""
    g = hub_batch(shape)
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    gen = torch.Generator().manual_seed(N + 1)
    h = torch.randn(N, 128, generator=gen)
    hd = h.to(DEV)
    L, st = lib(), _stream_ptr()
    ib = L.call("ddfa_act_image_bytes", N)
    h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_act_to_image", _p(hd), N, 128, _p(h_img), st)
    h_dec = decode_image(h_img, N)               # hi + lo: the exact values the image-to-image gather sums
    default = L.call("ddfa_tuning_get", TUNE_GATHER_SRC_GROUPS)
    worst = {}
    for orient, ip, ix, s_, d_ in _orientations(g, dg):
        ref, mag, deg = _gather_refs(h, s_, d_, N)
        s_img = torch.full((ib,), 0x55, dtype=torch.uint8, device=DEV)
        s_f = torch.full((N, 128), float("nan"), device=DEV)
        L.call("ddfa_gather_sum_image", _p(ip), _p(ix), _p(hd), N, 128, _p(s_img), _p(s_f), st)
        plain = torch.empty(N, 128, device=DEV)
        L.call("ddfa_gather_sum_variant", 0, _p(ip), _p(ix), _p(hd), N, 128, _p(plain), 0, st)
        assert torch.equal(s_f, plain), orient          # same neighbour order, same fp32 sums
        worst[f"{orient},f32"] = _ratio((s_f.cpu().double() - ref).abs(), 2 * deg * U * mag)
        sf64 = s_f.cpu().double()
        # the image holds hi + lo of each sum x: bf16 hi, then bf16 of x - hi, within 2^-17 |x| of it
        worst[f"{orient},image split"] = _ratio((decode_image(s_img, N) - sf64).abs(), 2.0 ** -17 * sf64.abs())
        ref_i, mag_i, _ = _gather_refs(h_dec, s_, d_, N)
        imgs = []
        try:
            for groups in (1, 2, 4):
                L.call("ddfa_tuning_set", TUNE_GATHER_SRC_GROUPS, groups)
                o = torch.full((ib,), 0x55, dtype=torch.uint8, device=DEV)
                L.call("ddfa_gather_sum_image_src", _p(ip), _p(ix), _p(h_img), N, 128, _p(o), st)
                imgs.append(o)
        finally:
            L.call("ddfa_tuning_set", TUNE_GATHER_SRC_GROUPS, default)
        assert torch.equal(imgs[1], imgs[0]) and torch.equal(imgs[2], imgs[0]), orient
        worst[f"{orient},image src"] = _ratio((decode_image(imgs[0], N) - ref_i).abs(), 2 * deg * U * mag_i + 2.0 ** -17 * ref_i.abs())
    print(f"image gathers, {shape} N={N}: worst |err| / bound: " + ", ".join(f"{k}={v:.2f}" for k, v in worst.items()))
    assert max(worst.values()) <= 1.0, worst


# ---------------------------------------------------------------------------------------------
def _gru_reference(s, h, deg, wf, bf, bih, whh, bhh):
    D_ = h.shape[1]
    gi = s @ wf.t() + deg[:, None] * bf[None, :] + bih
    gh = h @ whh.t() + bhh
    r = torch.sigmoid(gi[:, :D_] + gh[:, :D_]); z = torch.sigmoid(gi[:, D_:2 * D_] + gh[:, D_:2 * D_])
    n = torch.tanh(gi[:, 2 * D_:] + r * gh[:, 2 * D_:])
    return (1 - z) * n + z * h, r, z, n, gh[:, 2 * D_:]


GRAD_NAMES = ("dwf", "dbf", "dbih", "dwhh", "dbhh")


@pytest.mark.parametrize("shape", ["threshold", "c1"])
def test_tc_step_fwd_bwd_at_scale(shape):
    """One tensor-core GRU step (gru_fwd3_kernel; gate backward, dgrad3_kernel, wgrad_kernel) on the image entry points, at the
    gate backward's refill threshold and at C1 size, against fp64 autograd of the same math — test_gru_step_image_entries_v2
    at scale, with the gate backward in all three modes and the h operand as the image and as fp32 rows."""
    D_ = 128
    g = hub_batch(shape)
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    src, dst = g.edges()
    torch.manual_seed(N)
    k = 1.0 / D_ ** 0.5
    mk = lambda *sh: (torch.rand(*sh, dtype=torch.float64) * 2 - 1) * k
    wf, bf, bih, whh, bhh = mk(3 * D_, D_) * 1.5, mk(3 * D_), mk(3 * D_), mk(3 * D_, D_), mk(3 * D_)
    L, st = lib(), _stream_ptr()
    ib = L.call("ddfa_act_image_bytes", N)
    h32 = torch.tanh(torch.randn(N, D_)).to(DEV)
    h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_act_to_image", _p(h32), N, D_, _p(h_img), st)
    h = decode_image(h_img, N)
    deg = torch.bincount(dst, minlength=N).double()
    dh_part = torch.randn(N, D_, dtype=torch.float64)
    ds_prev = torch.randn(N, D_, dtype=torch.float64)
    leaves = [t.requires_grad_(True) for t in (h, wf, bf, bih, whh, bhh)]
    s_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gather_sum_image_src", _p(dg.indptr), _p(dg.indices), _p(h_img), N, D_, _p(s_img), st)
    s_leaf = decode_image(s_img, N).requires_grad_(True)       # the forward step consumes exactly this image
    h_ref, r_ref, z_ref, n_ref, ghn_ref = _gru_reference(s_leaf, leaves[0], deg, *leaves[1:])
    dh_in = dh_part + torch.zeros(N, D_, dtype=torch.float64).index_add(0, src, ds_prev[dst])
    (h_ref * dh_in).sum().backward()
    wfd, bfd, bihd, whhd, bhhd = [t.detach().float().to(DEV) for t in leaves[1:]]
    worst = {}

    # forward: image out + packed gates (middle step), fp32 out (last step), fp32 h operand (first step)
    wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D_, ENGINE_TCGEN05)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare", _p(wfd), _p(bfd), _p(bihd), _p(whhd), _p(bhhd), D_, ENGINE_TCGEN05, _p(ws), wsb, st)
    gates = torch.empty(L.call("ddfa_gru_gates_packed_bytes", N, D_), dtype=torch.uint8, device=DEV)
    o_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D_, None, _p(o_img), _p(gates), _p(ws), wsb, st)
    worst["h' image"] = float((decode_image(o_img, N) - h_ref.detach()).abs().max())
    for name, got, ref in zip(("r", "z", "n", "gh_n"), decode_gates(gates, N), (r_ref, z_ref, n_ref, ghn_ref)):
        scale = max(1.0, float(ref.abs().max())) if name == "gh_n" else 1.0
        worst[name] = float((got - ref.detach()).abs().max()) / scale
    h_out = torch.empty(N, D_, device=DEV)
    L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D_, _p(h_out), None, None, _p(ws), wsb, st)
    worst["h' fp32"] = float((h_out.cpu().double() - h_ref.detach()).abs().max())
    o_img2 = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_act_to_image", _p(h_out), N, D_, _p(o_img2), st)
    assert torch.equal(o_img, o_img2)
    h_out0 = torch.empty(N, D_, device=DEV)
    L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), _p(h32), _p(dg.indptr), N, D_, _p(h_out0), None, None, _p(ws), wsb, st)
    assert float((h_out0 - h_out).abs().max()) < 2e-5

    # backward from the image + packed gates, transposed gather folded in: gate backward modes 2 (default), 1, 0 x h operand forms
    wsb_b = L.call("ddfa_gru_step_bwd_workspace_bytes", N, D_, ENGINE_TCGEN05)
    ws_b = torch.empty(wsb_b, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare_bwd", _p(wfd), _p(whhd), D_, ENGINE_TCGEN05, _p(ws_b), wsb_b, st)
    dpart_d, dsprev_d = dh_part.float().to(DEV), ds_prev.float().to(DEV)
    refs = dict(ds=s_leaf.grad, dh=leaves[0].grad, dwf=wf.grad, dbf=bf.grad, dbih=bih.grad, dwhh=whh.grad, dbhh=bhh.grad)
    default = L.call("ddfa_tuning_get", TUNE_GATE_BWD_TMA)
    outs = {}
    try:
        for mode in (2, 1, 0):
            L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, mode)
            for h_arg in (None, _p(h32)):
                got = dict(ds=torch.full((N, D_), float("nan"), device=DEV), dh=torch.full((N, D_), float("nan"), device=DEV))
                got.update({n_: torch.zeros_like(refs[n_], dtype=torch.float32, device=DEV) for n_ in GRAD_NAMES})
                L.call("ddfa_gru_step_bwd_image_v2", _p(dpart_d), _p(dsprev_d), _p(dg.indptr_t), _p(dg.indices_t), h_arg, _p(h_img),
                       _p(s_img), _p(gates), _p(dg.indptr), N, D_, _p(got["ds"]), _p(got["dh"]), *[_p(got[n_]) for n_ in GRAD_NAMES],
                       _p(ws_b), wsb_b, 0, st)
                torch.cuda.synchronize()
                outs[(mode, h_arg is None)] = got
    finally:
        L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, default)
    for key, got in outs.items():
        for n_, ref in refs.items():
            err = float((got[n_].cpu().double() - ref).abs().max()) / max(1.0, float(ref.abs().max()))
            worst[n_] = max(worst.get(n_, 0.0), err)
    for key in ((2, True), (2, False), (1, True), (1, False)):
        a, b = outs[key], outs[(0, key[1])]
        assert torch.equal(a["ds"], b["ds"]) and torch.equal(a["dh"], b["dh"]), key
        for n_ in ("dbf", "dbih", "dbhh"):
            assert (a[n_] - b[n_]).abs().max() < 1e-4 * max(1.0, float(b[n_].abs().max())), (key, n_)
    print(f"tc step, {shape} N={N}: worst |err| (h', r, z, n absolute; gh_n and gradients / max(1, |ref|max)): "
          + ", ".join(f"{k_}={v:.1e}" for k_, v in worst.items()))
    bounds = {"h' image": 1e-4, "h' fp32": 1e-4, "r": 1.5e-4, "z": 1.5e-4, "n": 1.5e-4, "gh_n": 1.5e-4}
    bad = {k_: v for k_, v in worst.items() if v >= bounds.get(k_, 3e-4)}
    assert not bad, bad


# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [8, 17])
def test_ggnn_fused_drivers_at_scale(T):
    """ddfa_ggnn_fwd / ddfa_ggnn_bwd (the whole GatedGraphConv) on a 40 000-node hub batch, both engines, against fp64 autograd of
    the oracle's restatement.  T = 8 runs the batched weight gradient (about 113 tiles per wgrad CTA); T = 17 the per-step deferred
    accumulation closed by ddfa_gru_step_bwd_finish.  Bounds of test_kernels_gpu.py::test_ggnn_fused_drivers."""
    D_ = 128
    g = hub_batch("mid")
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    torch.manual_seed(T)
    conv = O.GatedGraphConvRestated(D_, D_, T).double()
    with torch.no_grad():
        conv.linears[0].bias.uniform_(-0.2, 0.2)          # DGL initialises it to zero; exercise the bias path
    x = (torch.randn(N, D_, dtype=torch.float64) * 0.5).requires_grad_(True)
    h_ref = conv(g, x)
    dh_T = torch.randn(N, D_, dtype=torch.float64)
    (h_ref * dh_T).sum().backward()
    par = dict(w_msg=conv.linears[0].weight, b_msg=conv.linears[0].bias, w_ih=conv.gru.weight_ih, w_hh=conv.gru.weight_hh,
               b_ih=conv.gru.bias_ih, b_hh=conv.gru.bias_hh)
    pd = {k: v.detach().float().to(DEV) for k, v in par.items()}
    xd, dhd = x.detach().float().to(DEV), dh_T.float().to(DEV)
    # s_v sums the h rows of v's in-neighbours, so their independent rounding errors grow like sqrt(in-degree) in it: the forward
    # bound (made on batches whose in-degrees stay below about 16) scales with sqrt(deg / 16) at the hubs.  Measured at the
    # 1100-neighbour hub, T = 8: both engines 7.5x their largest error on the rows of in-degree <= 16
    amp = (torch.bincount(g.edges()[1], minlength=N).double() / 16).sqrt().clamp_min(1.0)[:, None]
    L, st = lib(), _stream_ptr()
    worst = {}
    for engine in (ENGINE_SIMT, ENGINE_TCGEN05):
        name = "simt" if engine == ENGINE_SIMT else "tc"
        wsb = L.call("ddfa_ggnn_workspace_bytes", N, D_, T, engine, 1)
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
        h_out = torch.full((N, D_), float("nan"), device=DEV)
        L.call("ddfa_ggnn_fwd", _p(dg.indptr), _p(dg.indices), _p(xd), N, D_, T, _p(pd["w_msg"]), _p(pd["b_msg"]), _p(pd["w_ih"]),
               _p(pd["w_hh"]), _p(pd["b_ih"]), _p(pd["b_hh"]), _p(h_out), _p(ws), wsb, 1, engine, st)
        tol = (3e-5 if engine == ENGINE_SIMT else 2e-4) * T
        worst[f"{name} h_T"] = float(((h_out.cpu().double() - h_ref.detach()).abs() / amp).max()) / tol
        dx = torch.full((N, D_), float("nan"), device=DEV)
        gr = {k: torch.zeros_like(v) for k, v in pd.items()}
        L.call("ddfa_ggnn_bwd", _p(dg.indptr), _p(dg.indptr_t), _p(dg.indices_t), _p(xd), N, D_, T, _p(pd["w_msg"]), _p(pd["b_msg"]),
               _p(pd["w_ih"]), _p(pd["w_hh"]), _p(dhd), _p(dx), _p(gr["w_msg"]), _p(gr["b_msg"]), _p(gr["w_ih"]), _p(gr["w_hh"]),
               _p(gr["b_ih"]), _p(gr["b_hh"]), _p(ws), wsb, engine, st)
        gtol = (1e-4 if engine == ENGINE_SIMT else 5e-4) * T ** 0.5
        for k, got, ref in [("dx", dx, x.grad)] + [(k, gr[k], par[k].grad) for k in par]:
            worst[f"{name} {k}"] = float((got.cpu().double() - ref).abs().max()) / (gtol * max(1.0, float(ref.abs().max())))
    print(f"ggnn drivers, N={N} T={T}: worst |err| / bound: " + ", ".join(f"{k}={v:.2f}" for k, v in worst.items()))
    assert max(worst.values()) < 1.0, worst


# ---------------------------------------------------------------------------------------------
# per-parameter gradient bound relative to the largest entry of that parameter's reference gradient, as in
# test_parity_gpu.py::test_full_size_gradients_against_live_oracle
GRAD_TOL = {"simt": 1e-5, "tcgen05": 1e-4}
# bound on the proportional bias of the GGNN weight gradients; before the weight-gradient kernel summed its tiles with
# round-to-nearest adds, it was -1.0e-4 .. -1.2e-4 here (tensor-core engine)
BETA_TOL = 1e-5


@pytest.fixture(scope="module")
def c1_oracle():
    g = synth.make_batch(**MODULE_C1)
    torch.manual_seed(1)
    o = O.OracleFlowGNNGGNN(FEAT, 1002, 32, 8, 3, concat_all_absdf=True, positive_weight=4.0).double()
    loss_ref, _ = o.training_loss(g)
    loss_ref.backward()
    return g, o, float(loss_ref)


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_module_gradients_at_c1(c1_oracle, engine):
    """The production training step's gradients end to end at the size the benchmark runs (1024 graphs, 157 377 nodes, T = 8):
    embedding backward over every row, readout backward, the gate backward ring, the batched weight gradient."""
    g, o, loss_ref = c1_oracle
    m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 3, concat_all_absdf=True, positive_weight=4.0, engine=engine)
    m.load_state_dict({k: v.float() for k, v in o.state_dict().items()})
    m.to(DEV)
    loss = m.training_step((g.to(DEV), {}), 0)
    loss.backward()
    worst, shrink = {}, {}
    for (name, p), (_, q) in zip(m.named_parameters(), o.named_parameters()):
        ref, got = q.grad, p.grad.cpu().double()
        scale = max(float(ref.abs().max()), 1e-3)       # pooling.gate_nn.bias: true gradient 0 (softmax shift invariance)
        worst[name] = float((got - ref).abs().max()) / scale
        # a proportional bias, got = (1 + beta) ref, is what a biased accumulation over many tiles leaves behind
        shrink[name] = float(((got - ref) * ref).sum() / (ref * ref).sum().clamp_min(1e-300))
    print(f"module gradients at C1 (N={g.num_nodes()}), engine={engine}: |dloss|={abs(float(loss) - loss_ref):.1e}; worst per parameter: "
          + ", ".join(f"{k}={v:.1e}" for k, v in worst.items()) + "; beta of the GGNN weights: "
          + ", ".join(f"{k}={v:+.1e}" for k, v in shrink.items() if k.startswith("ggnn.")))
    assert abs(float(loss) - loss_ref) < 1e-4
    bad = {k: v for k, v in worst.items() if v >= GRAD_TOL[engine]}
    assert not bad, bad
    biased = {k: v for k, v in shrink.items() if k.startswith("ggnn.") and abs(v) >= BETA_TOL}
    assert not biased, biased
