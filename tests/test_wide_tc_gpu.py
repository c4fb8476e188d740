"""GPU: the tensor-core engine at hidden widths 192 .. 512 (csrc/gru_tc_wide.cu), against float64 references.

At these widths engine="tcgen05" keeps the SIMT engine's data flow and runs the six GEMMs of a GRU step on wgmma with bf16x3 split
operands.  Here each GEMM runs on its own at the C1 node count (157 381 nodes: ragged to 128 and to 64), then one GRU step on the
C1 hub batch, the whole GatedGraphConv (T = 8), the module's gradients, FusedTrainer and FusedEvaluator, and a 200-step run whose
decisions must follow the SIMT engine's.  Every test prints its worst error divided by its bound.

Bounds.  One bf16x3 product differs from the fp32 product by at most 3 * 2^-18 of |a b| (the dropped lo * lo term and the two
split remainders); the products are summed in fp32, 64 per MMA step (at most 3 * 64 roundings, with the tensor core's truncating
adds counted as one ulp, 2^-23), then one step at a time in fp32 and once more into C.  So a GEMM element is within
(2^-16 + (192 + K / 64 + 3) 2^-23) sum |a||b| (+ one rounding of |C_0|).  The step, GatedGraphConv and module bounds are the
D = 128 tensor-core bounds of tests/test_scale_gpu.py scaled by sqrt(W / 128), as tests/test_width_gpu.py scales the SIMT ones."""
import contextlib
import copy

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import synth
from deepdfa_b200._lib import ENGINE_TCGEN05, TUNE_DETERMINISTIC, lib
from deepdfa_b200 import engine as E
from deepdfa_b200.engine import _p, _stream_ptr, prepare_graph
from oracle import ggnn_oracle as O
from scale_batches import MODULE_C1, hub_batch
from test_scale_gpu import _gru_reference
from wide_tc_shapes import WIDE_WIDTHS, wgrad_slices
from width_batches import C1_NODES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
PAD = 37            # rows past N in every output buffer: they must keep their sentinel
SENTINEL = 7.0


def _wf(W):
    return max(1.0, (W / 128) ** 0.5)


@contextlib.contextmanager
def _mode(deterministic):
    L = lib()
    prev = L.call("ddfa_tuning_get", TUNE_DETERMINISTIC)
    L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, int(deterministic))
    try:
        yield
    finally:
        L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, prev)


def _report(title, worst):
    print(f"{title}: worst |err| / bound: " + ", ".join(f"{k}={v:.3f}" for k, v in worst.items()))


def _assert_within(worst):
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad


@pytest.fixture(autouse=True)
def _free_memory():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    yield


# ---- the six GEMM calls ---------------------------------------------------------------------------------------------------
BETA_TOL = 1e-5         # test_scale_gpu.py::BETA_TOL: proportional bias (got = (1 + beta) ref) of a whole result


def _beta(got, ref):
    """The proportional bias of got against ref: the least-squares beta of got - ref = beta ref."""
    return float(((got - ref) * ref).sum() / (ref * ref).sum().clamp_min(1e-300))


def _gemm_bound(mag, K, c0=None):
    b = (2.0 ** -16 + (192 + -(-K // 64) + 3) * 2.0 ** -23) * mag
    return b if c0 is None else b + 2.0 ** -24 * c0.double().abs()


@pytest.mark.parametrize("W", WIDE_WIDTHS)
def test_gemm_calls_at_c1(W):
    """The six GEMMs of one step through ddfa_gru_tc_wide_gemm at N = 157 381: gi = s W'^T, gh = h Whh^T, ds = dgi W',
    dh += dgh Whh, dW' += dgi^T s, dWhh += dgh^T h, against fp64 matmuls; rows past N keep their sentinel; the weight gradient is
    bit-identical on repeat in both modes."""
    N = C1_NODES
    L, st = lib(), _stream_ptr()
    gen = torch.Generator(device=DEV).manual_seed(W)
    k = W ** -0.5
    s = torch.randn(N, W, device=DEV, generator=gen) * 4
    h = torch.tanh(torch.randn(N, W, device=DEV, generator=gen))
    wf = (torch.rand(3 * W, W, device=DEV, generator=gen) * 2 - 1) * 1.5 * k
    whh = (torch.rand(3 * W, W, device=DEV, generator=gen) * 2 - 1) * k
    dgi = torch.randn(N, 3 * W, device=DEV, generator=gen) * 0.1
    dgh = torch.randn(N, 3 * W, device=DEV, generator=gen) * 0.1
    calls = [("gi", 0, s, wf), ("gh", 0, h, whh), ("ds", 1, dgi, wf), ("dh", 2, dgh, whh), ("dW'", 3, dgi, s), ("dWhh", 3, dgh, h)]
    worst = {}
    for i, (name, call, a, b) in enumerate(calls):
        wsb = L.call("ddfa_gru_tc_wide_gemm_workspace_bytes", call, N, W)
        ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)      # garbage: the call must not read unwritten workspace
        if call == 3:
            ref = a.double().t() @ b.double()
            mag = a.double().abs().t() @ b.double().abs()
            c0 = torch.randn(3 * W, W, device=DEV, generator=gen)
            outs = []
            for det in (False, True, True):
                with _mode(det):
                    c = c0.clone()
                    L.call("ddfa_gru_tc_wide_gemm", call, _p(a), _p(b), N, W, _p(c), _p(ws), wsb, st)
                    outs.append(c)
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2]), f"{name}: not bit-identical on repeat"
            got, bound = outs[0].double(), _gemm_bound(mag, N, c0)
            ref = ref + c0.double()
        else:
            ref = a.double() @ (b.double().t() if call == 0 else b.double())
            mag = a.double().abs() @ (b.double().abs().t() if call == 0 else b.double().abs())
            c = torch.full((N + PAD, ref.shape[1]), SENTINEL, device=DEV)
            c0 = None
            if call == 2:
                c0 = torch.randn(N, W, device=DEV, generator=gen)
                c[:N] = c0
                ref = ref + c0.double()
            L.call("ddfa_gru_tc_wide_gemm", call, _p(a), _p(b), N, W, _p(c), _p(ws), wsb, st)
            torch.cuda.synchronize()
            assert bool((c[N:] == SENTINEL).all()), f"{name}: a row past N was written"
            got, bound = c[:N].double(), _gemm_bound(mag, b.shape[0] if call else W, c0)
        worst[name] = float(((got - ref).abs() / bound).max())
        # a systematic relative shrink of the result (got = (1 + beta) ref) hides inside the worst-case bound: bounded on its own
        worst[f"{name} beta"] = abs(_beta(got, ref)) / BETA_TOL
        del ref, mag, got, bound
    sl = wgrad_slices(N, W)
    _report(f"wide gemm calls W={W} N={N} (weight gradient: {sl['nz']} slices of {sl['kps']} steps)", worst)
    _assert_within(worst)


# ---- one GRU step -----------------------------------------------------------------------------------------------------------
GRAD_NAMES = ("dwf", "dbf", "dbih", "dwhh", "dbhh")


@pytest.mark.parametrize("W", WIDE_WIDTHS)
def test_gru_step_at_c1(W):
    """ddfa_gru_step_fwd / _bwd on the tensor-core engine over the C1 hub batch (157 381 nodes): h', the four gate planes, ds, dh
    and the five weight / bias gradients against fp64 autograd of the same math, in default and deterministic mode (bit-identical
    over a garbage workspace); rows of h', ds, dh past N keep their sentinel.  Bounds of test_scale_gpu.py::
    test_tc_step_fwd_bwd_at_scale x sqrt(W / 128); the proportional bias of ds, dh and each gradient below BETA_TOL."""
    g = hub_batch("c1")
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    L, st = lib(), _stream_ptr()
    gen = torch.Generator(device=DEV).manual_seed(W)
    k = W ** -0.5
    mk = lambda *sh: ((torch.rand(*sh, device=DEV, generator=gen) * 2 - 1) * k)
    wf, bf, bih, whh, bhh = mk(3 * W, W) * 1.5, mk(3 * W), mk(3 * W), mk(3 * W, W), mk(3 * W)
    h32 = torch.tanh(torch.randn(N, W, device=DEV, generator=gen))
    s32 = torch.empty(N, W, device=DEV)
    L.call("ddfa_gather_sum", _p(dg.indptr), _p(dg.indices), _p(h32), N, W, _p(s32), 0, st)
    dh_out = torch.randn(N, W, device=DEV, generator=gen)
    deg = torch.bincount(g.edges()[1].to(DEV), minlength=N).double()
    leaves = [t.double().requires_grad_(True) for t in (s32, h32, wf, bf, bih, whh, bhh)]
    h_ref, *gate_refs = _gru_reference(leaves[0], leaves[1], deg, *leaves[2:])
    (h_ref * dh_out.double()).sum().backward()
    h_ref = h_ref.detach()
    gate_refs = [t.detach() for t in gate_refs]
    refs = dict(ds=leaves[0].grad, dh=leaves[1].grad, dwf=leaves[2].grad, dbf=leaves[3].grad, dbih=leaves[4].grad,
                dwhh=leaves[5].grad, dbhh=leaves[6].grad)
    del leaves
    wfac = _wf(W)
    tol = dict(h=1e-4 * wfac, gate=1.5e-4 * wfac, grad=3e-4 * wfac)
    wsb = L.call("ddfa_gru_step_workspace_bytes", N, W, ENGINE_TCGEN05)
    ws = torch.full((wsb,), 0xAB, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare", _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), W, ENGINE_TCGEN05, _p(ws), wsb, st)
    wsb_b = L.call("ddfa_gru_step_bwd_workspace_bytes", N, W, ENGINE_TCGEN05)
    ws_b = torch.empty(wsb_b, dtype=torch.uint8, device=DEV)
    worst, results = {}, {}
    for det in (False, True):
        mode = "det" if det else "default"
        with _mode(det):
            h_out = torch.full((N + PAD, W), SENTINEL, device=DEV)
            gates = torch.full((4, N, W), float("nan"), device=DEV)
            L.call("ddfa_gru_step_fwd", _p(s32), _p(h32), _p(dg.indptr), _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), N, W, _p(h_out),
                   _p(gates), _p(ws), wsb, ENGINE_TCGEN05, st)
            runs = []
            for rep in range(2 if det else 1):
                ws_b.fill_(0xAB)
                L.call("ddfa_gru_step_prepare_bwd", _p(wf), _p(whh), W, ENGINE_TCGEN05, _p(ws_b), wsb_b, st)
                got = dict(ds=torch.full((N + PAD, W), SENTINEL, device=DEV), dh=torch.full((N + PAD, W), SENTINEL, device=DEV))
                got.update({n_: torch.zeros_like(refs[n_], dtype=torch.float32) for n_ in GRAD_NAMES})
                L.call("ddfa_gru_step_bwd", _p(dh_out), _p(h32), _p(s32), _p(gates), _p(dg.indptr), _p(wf), _p(whh), N, W, _p(got["ds"]),
                       _p(got["dh"]), *[_p(got[n_]) for n_ in GRAD_NAMES], _p(ws_b), wsb_b, ENGINE_TCGEN05, st)
                runs.append(got)
            torch.cuda.synchronize()
        for t in (h_out, runs[0]["ds"], runs[0]["dh"]):
            assert bool((t[N:] == SENTINEL).all()), "a row past N was written"
        h_out = h_out[:N]
        if det:
            assert torch.equal(h_out, results["default"][0]) and torch.equal(gates, results["default"][1])
            assert all(torch.equal(runs[1][n_], runs[0][n_]) for n_ in refs), "deterministic backward not repeatable"
        else:
            worst["h'"] = float((h_out.double() - h_ref).abs().max()) / tol["h"]
            for name, got_, ref in zip(("r", "z", "n", "gh_n"), gates, gate_refs):
                scale = max(1.0, float(ref.abs().max())) if name == "gh_n" else 1.0
                worst[name] = float((got_.double() - ref).abs().max()) / (tol["gate"] * scale)
        for n_, ref in refs.items():
            got_ = runs[0][n_][:N] if n_ in ("ds", "dh") else runs[0][n_]
            worst[f"{n_} {mode}"] = float((got_.double() - ref).abs().max()) / (tol["grad"] * max(1.0, float(ref.abs().max())))
            if not det:
                worst[f"{n_} beta"] = abs(_beta(got_.double(), ref)) / BETA_TOL
        results[mode] = (h_out, gates)
        del runs
    _report(f"tc gru step W={W} N={N}", worst)
    _assert_within(worst)


# ---- whole GatedGraphConv -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", WIDE_WIDTHS)
def test_ggnn_drivers_at_width(W):
    """ddfa_ggnn_fwd / ddfa_ggnn_bwd on the tensor-core engine, T = 8, on the 40 001-node hub batch, against fp64 autograd of the
    oracle's GatedGraphConv restatement.  Bounds of test_scale_gpu.py::test_ggnn_fused_drivers_at_scale (tensor-core engine)
    x sqrt(W / 128), and the proportional bias of dx and of the weight matrices' gradients below BETA_TOL x sqrt(W / 128)."""
    T = 8
    g = hub_batch("mid")
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    torch.manual_seed(W)
    conv = O.GatedGraphConvRestated(W, W, T).double().to(DEV)
    with torch.no_grad():
        conv.linears[0].bias.uniform_(-0.2, 0.2)
        for p in conv.parameters():
            p.copy_(p.float().double())
    x = (torch.randn(N, W, device=DEV) * 0.5).double().requires_grad_(True)
    h_ref = conv(g.to(DEV), x)
    dh_T = torch.randn(N, W, device=DEV)
    (h_ref * dh_T.double()).sum().backward()
    par = dict(w_msg=conv.linears[0].weight, b_msg=conv.linears[0].bias, w_ih=conv.gru.weight_ih, w_hh=conv.gru.weight_hh,
               b_ih=conv.gru.bias_ih, b_hh=conv.gru.bias_hh)
    pd = {k: v.detach().float() for k, v in par.items()}
    xd = x.detach().float()
    amp = (torch.bincount(g.edges()[1].to(DEV), minlength=N).double() / 16).sqrt().clamp_min(1.0)[:, None]
    L, st = lib(), _stream_ptr()
    wsb = L.call("ddfa_ggnn_workspace_bytes", N, W, T, ENGINE_TCGEN05, 1)
    assert wsb > 0
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    h_out = torch.full((N, W), float("nan"), device=DEV)
    L.call("ddfa_ggnn_fwd", _p(dg.indptr), _p(dg.indices), _p(xd), N, W, T, _p(pd["w_msg"]), _p(pd["b_msg"]), _p(pd["w_ih"]),
           _p(pd["w_hh"]), _p(pd["b_ih"]), _p(pd["b_hh"]), _p(h_out), _p(ws), wsb, 1, ENGINE_TCGEN05, st)
    worst = {"h_T": float(((h_out.double() - h_ref.detach()).abs() / amp).max()) / (2e-4 * T * _wf(W))}
    dx = torch.full((N, W), float("nan"), device=DEV)
    gr = {k: torch.zeros_like(v) for k, v in pd.items()}
    L.call("ddfa_ggnn_bwd", _p(dg.indptr), _p(dg.indptr_t), _p(dg.indices_t), _p(xd), N, W, T, _p(pd["w_msg"]), _p(pd["b_msg"]),
           _p(pd["w_ih"]), _p(pd["w_hh"]), _p(dh_T), _p(dx), _p(gr["w_msg"]), _p(gr["b_msg"]), _p(gr["w_ih"]), _p(gr["w_hh"]),
           _p(gr["b_ih"]), _p(gr["b_hh"]), _p(ws), wsb, ENGINE_TCGEN05, st)
    gtol = 5e-4 * T ** 0.5 * _wf(W)
    # Proportional bias: dx and the three weight matrices within BETA_TOL x sqrt(W / 128).  The three bias vectors are reported:
    # here each of their entries is a sum over 40 001 nodes of random-sign terms that cancel 20x to 200x (sum |g| / |sum g|), and
    # their beta is the projection of the fp32 error of those sums, whose sign changes from width to width — the D = 128 tensor-
    # core engine gives -1.7e-5 to -2.8e-5 on this same test, the SIMT engine up to -8e-6 (H100 80GB HBM3, 700 W).  A systematic
    # shrink of the GGNN gradients is bounded where the gradient is a training signal: test_module_gradients_and_trainer_step.
    betas = {}
    for k, got, ref in [("dx", dx, x.grad)] + [(k, gr[k], par[k].grad) for k in par]:
        worst[k] = float((got.double() - ref).abs().max()) / (gtol * max(1.0, float(ref.abs().max())))
        if k.startswith("b_"):
            betas[k] = _beta(got.double(), ref)
        else:
            worst[f"{k} beta"] = abs(_beta(got.double(), ref)) / (BETA_TOL * _wf(W))
    print("bias-vector beta (reported): " + ", ".join(f"{k}={v:+.1e}" for k, v in betas.items()))
    _report(f"ggnn tc drivers W={W} N={N} T={T}", worst)
    _assert_within(worst)


# ---- the module, FusedTrainer and FusedEvaluator --------------------------------------------------------------------------
GRAD_TOL = 1e-4         # test_scale_gpu.py::GRAD_TOL["tcgen05"], per parameter, relative to its largest reference entry
# W -> (hidden_dim with concat_all_absdf, batch): C1 at W = 256; the 40 001-node hub batch (in-degrees up to 1100) at W = 192 (3W
# and W end on a half tile) and at W = 512, where tests/test_width_gpu.py holds the SIMT engine
MODULE_WIDTHS = {192: (48, "mid"), 256: (64, "c1"), 512: (128, "mid")}


def _kernel_relu_masks(m, gd):
    """Which units of the MLP's hidden layers the kernels' forward passes (pre-activation > 0), [B, 2W] per hidden layer: the
    same forward kernels as the training step, run through engine.forward, with the saved post-ReLU activations read back."""
    _, dg, idx = m._prepare(gd)
    params = E.ParamPack.from_flat_list([t.detach() for t in m.param_list()], len(m._tables()), m._num_layers)
    _, _, saved = E.forward(params, dg, idx, m.hparams.n_steps, training=True, engine=ENGINE_TCGEN05)
    return [a > 0 for a in saved.mlp_act]


def _oracle_on_kernel_side(o, g, masks):
    """The float64 loss and gradients of the oracle with each hidden ReLU evaluated on the side of its kink the kernels took.

    The MLP head is piecewise linear, so its gradient jumps where a pre-activation crosses 0.  A few of the C1 / hub-batch units
    sit within 1e-7 of 0 (e.g. 8 of 259 072 below 1e-5 at W = 512 on the hub batch), closer than any fp32 forward's error (the
    tensor-core forward's logits differ from fp64 by about 5e-7), and a unit that lands on the other side changes the gradient of
    everything below it by O(its weight) — a difference of the reference's branch, not an error of the kernels.  So the reference
    is taken on the kernels' branch: relu(x) becomes x * mask, identical to relu wherever the two sides agree.  Returns the loss
    and the number of units where the float64 forward and the kernels disagree."""
    relus = [mod for mod in o.output_layer if isinstance(mod, torch.nn.ReLU)]
    assert len(relus) == len(masks)
    flips = [0]

    def hook(mod, inp, out, mk):
        flips[0] += int(((inp[0] > 0) != mk).sum())
        return inp[0] * mk.to(inp[0].dtype)
    handles = [r.register_forward_hook(lambda mod, inp, out, mk=mk: hook(mod, inp, out, mk)) for r, mk in zip(relus, masks)]
    try:
        loss_ref, _ = o.training_loss(g)
        loss_ref.backward()
    finally:
        for h_ in handles:
            h_.remove()
    return float(loss_ref), flips[0]


def _module(hidden, o, engine="tcgen05", **kw):
    m = D.FlowGNNGGNNModule(FEAT, 1002, hidden, 8, 3, concat_all_absdf=True, positive_weight=4.0, engine=engine, **kw)
    m.load_state_dict({k: v.float().cpu() for k, v in o.state_dict().items()})
    return m.to(DEV)


@pytest.mark.parametrize("W", list(MODULE_WIDTHS))
def test_module_gradients_and_trainer_step(W):
    """The training step's loss and every parameter gradient against OracleFlowGNNGGNN in float64 (T = 8, three output layers;
    C1 batch at W = 256, the 40 001-node hub batch at W = 192 and 512), each within GRAD_TOL x sqrt(W / 128) of its largest
    reference entry and with a proportional bias of the GGNN weight gradients below BETA_TOL; then one FusedTrainer step against
    torch.optim.Adam on the oracle's gradients (the rule of tests/test_width_gpu.py::test_module_gradients_at_width).  The
    oracle's hidden ReLUs take the kernels' side of their kinks (_oracle_on_kernel_side)."""
    hidden, batch = MODULE_WIDTHS[W]
    g = synth.make_batch(**MODULE_C1) if batch == "c1" else hub_batch("mid")
    gd = g.to(DEV)
    torch.manual_seed(1)
    o = O.OracleFlowGNNGGNN(FEAT, 1002, hidden, 8, 3, concat_all_absdf=True, positive_weight=4.0).double().to(DEV)
    with torch.no_grad():
        for p in o.parameters():
            p.copy_(p.float().double())
    m = _module(hidden, o)
    assert m.engine == "tcgen05" and m._D == W
    loss_ref, flips = _oracle_on_kernel_side(o, gd, _kernel_relu_masks(m, gd))
    loss_t = m.training_step((gd, {}), 0)
    loss_t.backward()
    tol = GRAD_TOL * _wf(W)
    worst, shrink, delta = {}, {}, {}
    for (name, p), (_, q) in zip(m.named_parameters(), o.named_parameters()):
        ref, got = q.grad, p.grad.double()
        scale = max(float(ref.abs().max()), 1e-3)
        worst[name] = float((got - ref).abs().max()) / (tol * scale)
        shrink[name] = float(((got - ref) * ref).sum() / (ref * ref).sum().clamp_min(1e-300))
        delta[name] = tol * scale
    assert abs(float(loss_t) - loss_ref) < 1e-4
    biased = {k: v for k, v in shrink.items() if k.startswith("ggnn.") and abs(v) >= BETA_TOL}
    del m
    m2 = _module(hidden, o)
    tr = D.FusedTrainer(m2)
    lr, wd = tr.lr, tr.weight_decay
    loss_tr = float(tr.step(gd))
    p0 = {k: q.detach().clone() for k, q in o.named_parameters()}
    torch.optim.Adam(o.parameters(), lr=lr, weight_decay=wd).step()
    U = 2.0 ** -24
    for (name, p), (_, q) in zip(m2.named_parameters(), o.named_parameters()):
        gp = (q.grad + wd * p0[name]).abs()
        dl = delta[name]
        allowed = lr * torch.where(gp > 2 * dl, 2 * dl / gp.clamp_min(1e-300), torch.full_like(gp, 2.0)) + 2 * U * p0[name].abs() + 8 * U * lr
        worst[f"adam {name}"] = float(((p.detach().double() - q.detach()).abs() / allowed).max())
    _report(f"tc module gradients + trainer step W={W} N={g.num_nodes()} ({flips} ReLU units on the other side of their kink in "
            "fp64); beta: " + ", ".join(f"{k}={v:+.1e}" for k, v in shrink.items() if k.startswith("ggnn.")), worst)
    assert abs(loss_tr - loss_ref) < 1e-4
    assert not biased, biased
    _assert_within(worst)


def f1_at_half(prob, label):
    from sklearn.metrics import f1_score
    return float(f1_score(label.astype(int), (prob > 0.5).astype(int), zero_division=0))


def test_training_run_follows_the_simt_engine():
    """200 FusedTrainer steps at W = 256 (hidden_dim 64, concat_all_absdf) of both engines on one synthetic stream from the same
    weights, then both classify the same 768 held-out graphs: the decisions and the F1 at 0.5 must follow the SIMT engine's
    (the rule of tests/test_trainer_gpu.py::test_training_decisions_and_f1_follow_the_oracle)."""
    torch.manual_seed(0)
    ref = D.FlowGNNGGNNModule(FEAT, 1002, 64, 8, 2, concat_all_absdf=True, positive_weight=1.5, engine="simt")
    state = copy.deepcopy(ref.state_dict())
    stream = [synth.make_learnable_batch(24, 40, seed=300 + i) for i in range(40)]
    held = [synth.make_learnable_batch(256, 40, seed=900 + i) for i in range(3)]
    out = {}
    for engine in ("simt", "tcgen05"):
        m = D.FlowGNNGGNNModule(FEAT, 1002, 64, 8, 2, concat_all_absdf=True, positive_weight=1.5, engine=engine)
        m.load_state_dict(state)
        m.to(DEV)
        tr = D.FusedTrainer(m)
        losses = [float(tr.step(stream[i % len(stream)])) for i in range(200)]
        probs, labels = [], []
        with torch.no_grad():
            for b in held:
                _, p, lab = m.validation_step((b, {}), 0)
                probs.append(p.cpu().numpy())
                labels.append(lab.cpu().numpy())
        out[engine] = (losses, np.concatenate(probs), np.concatenate(labels))
    (ls, ps, y), (lt, pt, y2) = out["simt"], out["tcgen05"]
    assert np.array_equal(y, y2)
    agree = float(((ps > 0.5) == (pt > 0.5)).mean())
    f1_s, f1_t = f1_at_half(ps, y), f1_at_half(pt, y)
    print(f"train 200 steps W=256: loss simt {ls[0]:.4f} -> {ls[-1]:.4f}, tcgen05 {lt[0]:.4f} -> {lt[-1]:.4f}; held-out 768 graphs: "
          f"decision agreement {agree:.4f}, F1 simt {f1_s:.4f} vs tcgen05 {f1_t:.4f}, max|dprob| {float(np.abs(ps - pt).max()):.2e}")
    assert ls[-1] < 0.7 * ls[0], "the stream is learnable: the loss must fall"
    assert f1_s > 0.8, "the SIMT arm must have learned the task for the comparison to mean anything"
    assert agree >= 0.99 and abs(f1_s - f1_t) <= 0.02


def _trainer_state(tr, losses):
    return [p.detach().clone() for p in tr.module.parameters()], losses


def test_trainer_features_and_deterministic_runs():
    """At W = 256: FusedTrainer in deterministic mode twice from the same weights (graph style, a captured step, gradient
    accumulation over two micro-batches and the gradient guard) is bit-identical; node style, frozen parameters and the
    dgrad-only backward of FusedEvaluator(statements="saliency") agree with the SIMT engine."""
    batches = [synth.make_batch(128, 60, seed=40 + i, variable=True, vuln_rate=0.3) for i in range(4)]
    torch.manual_seed(3)
    base = D.FlowGNNGGNNModule(FEAT, 1002, 64, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine="simt")
    state = copy.deepcopy(base.state_dict())

    def make(engine, **kw):
        m = D.FlowGNNGGNNModule(FEAT, 1002, 64, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine, **kw)
        m.load_state_dict(state, strict=kw.get("label_style", "graph") == "graph")
        return m.to(DEV)

    import os
    prev = os.environ.get("DDFA_DETERMINISTIC")
    os.environ["DDFA_DETERMINISTIC"] = "1"
    try:
        runs = []
        for _ in range(2):
            tr = D.FusedTrainer(make("tcgen05"), use_cuda_graph=True, accumulate_grad_batches=2, max_grad_norm=1.0, skip_nonfinite=True)
            runs.append(_trainer_state(tr, [float(tr.step(batches[i % 4])) for i in range(6)]))
    finally:
        if prev is None:
            os.environ.pop("DDFA_DETERMINISTIC")
        else:
            os.environ["DDFA_DETERMINISTIC"] = prev
    assert runs[0][1] == runs[1][1] and all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0])), "deterministic runs differ"

    worst = {}
    # node style and frozen parameters: a few steps of both engines, loss by loss
    for label, kw, freeze in (("node", dict(label_style="node"), False), ("frozen tables", {}, True)):
        losses = {}
        for engine in ("simt", "tcgen05"):
            m = make(engine, **kw)
            if freeze:
                for n_, p in m.named_parameters():
                    if n_.startswith("all_embeddings."):      # the full GGNN backward without the embedding backward
                        p.requires_grad_(False)
            tr = D.FusedTrainer(m)
            losses[engine] = np.array([float(tr.step(batches[i])) for i in range(4)])
        worst[label] = float(np.abs(losses["simt"] - losses["tcgen05"]).max() / np.abs(losses["simt"]).max()) / 1e-3
    # the evaluator's dgrad-only backward: saliency scores of both engines
    scores = {}
    for engine in ("simt", "tcgen05"):
        ev = D.FusedEvaluator(make(engine), statements="saliency")
        ev.update(batches[0])
        torch.cuda.synchronize()
        scores[engine] = ev.last_scores().clone().double()
        assert "test_stmt_functions" in ev.compute("test_")
    # test_statements_gpu.py::GRAD_TOL["tcgen05"] (relative to the largest score) x sqrt(W / 128)
    worst["saliency"] = float((scores["simt"] - scores["tcgen05"]).abs().max() / scores["simt"].abs().max()) / (2e-3 * _wf(256))
    _report("tc W=256 trainer features vs simt (relative: 1e-3 of the loss, 2.8e-3 of the largest score)", worst)
    _assert_within(worst)
