"""GPU: the statement and attribution kernels of csrc/statements.cu, each called directly, at the edges of their launch shapes:
ddfa_stmt_attention (functions of 1 and 40 000 nodes, underflowing terms) against a float64 softmax; ddfa_stmt_input_grad_score
(both rules, D = 4 .. 512, N not a multiple of 8, accumulated passes) against float64; ddfa_stmt_attribution_score bit-identical
to the x * g rule; ddfa_stmt_scale_input and its activation image exactly; ddfa_stmt_shap_input over 3 000 functions (the grid
strides) against the host Philox of tests/attribution_rule.py; ddfa_stmt_node_probability for every clamp of its row count; and
ddfa_stmt_metric against tests/statement_rule.py::host_state, exactly, on ties across warps and iterations, signed zeros,
infinities and NaN, with more functions than CTAs.  Then FusedEvaluator's saliency, integrated-gradient and DeepLift scores on
the wide tensor-core engine (W = 192, 512) against the float64 oracle.  Every float comparison prints its worst error / bound."""
import contextlib
import math

import numpy as np
import pytest
import torch

import attribution_rule as A
import head_batches as H
import statement_rule as R
import deepdfa_b200 as D
from deepdfa_b200 import _lib
from deepdfa_b200.engine import _p, _stream_ptr
from oracle import ggnn_oracle as O
from scale_batches import HUB_SHAPES, hub_batch
from test_head_gpu import _readout_fwd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = 7.0
PAD = 37                # elements past N in every output buffer: they must keep their sentinel
U = H.U
HUB_NODES = HUB_SHAPES["mid"][2]


def _lib_call(name, *args):
    _lib.lib().call(name, *args)
    torch.cuda.synchronize()


def _report(title, worst):
    print(f"{title}: worst |err| / bound: " + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad


# ---- attention -------------------------------------------------------------------------------------------------------------
def test_attention_softmax_over_1_to_40000_nodes():
    """ddfa_stmt_attention from the readout's own gate logits, segment max and sum (ddfa_readout_mlp_fwd on graphs of 0, 1 and
    40 000 nodes, logits spread so that a third of the large graph's terms underflow) against float64 softmax of the same
    logits.  Bound per node: expf of the rounded difference gl - M ((|gl - M| + 4) u), the division (2 u) and the error of the
    readout's fp32 sum (head_batches.seg_sum_ref), plus the subnormal rounding; each function's alphas sum to 1 within the sum
    of their bounds (and 2 u per term)."""
    sizes = H.big_sizes()
    Dm = 32
    h, x, w, b = H.readout_inputs(sizes, Dm, seed=41, extreme=True)
    gp = H.graph_ptr(sizes).to(DEV)
    out = _readout_fwd(h.to(DEV), x.to(DEV), gp, sizes, Dm, w.to(DEV), b.to(DEV), [], [], 0)
    gl, smax, ssum = out["gl"], out["smax"], out["ssum"]
    N, B = len(gl), len(sizes)
    alpha = torch.full((N + PAD,), SENTINEL, device=DEV)
    gld, smd, ssd = gl.to(DEV), smax.to(DEV), ssum.to(DEV)
    _lib_call("ddfa_stmt_attention", _p(gld), _p(smd), _p(ssd), _p(gp), B, _p(alpha), _stream_ptr())
    assert bool((alpha[N:] == SENTINEL).all())
    got = alpha[:N].cpu().double()
    seg = H.segment_ids(sizes)
    d = gl.double() - smax.double()[seg]
    S_ref, S_bound = H.seg_sum_ref(gl, smax, sizes)
    ref = torch.exp(d) / S_ref[seg]
    bound = ref * ((d.abs() + 6) * U + (S_bound / S_ref)[seg]) + 4 * H.ETA     # expf within a subnormal spacing or two
    sums = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, got)
    sum_bound = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, bound + 2 * U * got)
    nonempty = torch.from_numpy(sizes > 0)
    big = int(np.argmax(sizes))
    under = int((got[seg == big] == 0).sum())
    assert under > sizes[big] // 4, "the large graph's logits must spread far enough to underflow"
    _report(f"stmt attention, graphs of 0 .. {sizes.max()} nodes ({under} alphas underflow to 0)",
            dict(alpha=H.ratio((got - ref).abs(), bound), sum=H.ratio((sums - 1).abs()[nonempty], sum_bound[nonempty])))


# ---- input-gradient scores --------------------------------------------------------------------------------------------------
def _score(rule, x, dh, dx, w, acc, score):
    N, Dm = dh.shape
    _lib_call("ddfa_stmt_input_grad_score", _p(x), _p(dh), _p(dx), N, Dm, rule, float(w), int(acc), _p(score), _stream_ptr())


@pytest.mark.parametrize("Dm", R.SCORE_WIDTHS)
def test_input_grad_score_both_rules(Dm):
    """Both rules (sum_d |dh + dx| and sum_d x (dh + dx)) at N = 40 001 (not a multiple of 8): one overwriting pass, then m = 3
    accumulated passes with weights onto a nonzero start, against float64.  Bound: ceil(D / 32) strided terms per lane, the
    5-level shuffle tree, dh + dx and the product (2 (ceil(D / 32) + 7) u of the magnitude), and one rounding of the running
    score per pass; attribution_score with diff in place of x is the x * g rule bit for bit."""
    N = HUB_NODES
    gen = torch.Generator(device=DEV).manual_seed(Dm)
    x = torch.randn(N, Dm, device=DEV, generator=gen)
    passes = [(torch.randn(N, Dm, device=DEV, generator=gen), torch.randn(N, Dm, device=DEV, generator=gen), w)
              for w in (1.0, 0.375, -2.5)]
    start = torch.randn(N, device=DEV, generator=gen)
    worst = {}
    for rule, name in ((_lib.STMT_SCORE_ABS, "abs"), (_lib.STMT_SCORE_X_TIMES, "x*g")):
        f = (lambda g: g.abs()) if rule == _lib.STMT_SCORE_ABS else (lambda g: x.double() * g)
        fm = (lambda g: g) if rule == _lib.STMT_SCORE_ABS else (lambda g: x.double().abs() * g)
        depth = 2 * (-(-Dm // 32) + 7) * U
        # one overwriting pass over a NaN start
        dh, dx, w = passes[1]
        score = torch.full((N + PAD,), float("nan"), device=DEV)
        score[N:] = SENTINEL
        _score(rule, x, dh, dx, w, False, score)
        g64, gm = dh.double() + dx.double(), dh.double().abs() + dx.double().abs()
        ref, mag = w * f(g64).sum(1), abs(w) * fm(gm).sum(1)
        worst[f"{name} set"] = H.ratio((score[:N].double() - ref).abs(), depth * mag)
        assert bool((score[N:] == SENTINEL).all())
        # m accumulated passes onto the start
        score = torch.cat([start, torch.full((PAD,), SENTINEL, device=DEV)])
        ref, mag = start.double().clone(), start.double().abs()
        for dh, dx, w in passes:
            _score(rule, x, dh, dx, w, True, score)
            g64, gm = dh.double() + dx.double(), dh.double().abs() + dx.double().abs()
            ref += w * f(g64).sum(1)
            mag += abs(w) * fm(gm).sum(1)
        worst[f"{name} accumulate"] = H.ratio((score[:N].double() - ref).abs(), (depth + 2 * len(passes) * U) * mag)
        assert bool((score[N:] == SENTINEL).all())
        if rule == _lib.STMT_SCORE_X_TIMES:
            other = torch.cat([start, torch.full((PAD,), SENTINEL, device=DEV)])
            for dh, dx, w in passes:
                _lib_call("ddfa_stmt_attribution_score", _p(x), _p(dh), _p(dx), N, Dm, float(w), 1, _p(other), _stream_ptr())
            assert torch.equal(other, score), "attribution_score is not the x * g rule bit for bit"
    _report(f"stmt input-grad score D={Dm} N={N}", worst)


def test_scale_input_and_its_image():
    """ddfa_stmt_scale_input: out = fp32(alpha x) exactly (one rounding, as torch's product), at D = 128 with the activation image
    equal to ddfa_act_to_image of the scaled rows, and at D = 20 without one."""
    for Dm, N in ((128, HUB_NODES), (20, 1001)):
        x = torch.randn(N, Dm, device=DEV, generator=torch.Generator(device=DEV).manual_seed(N))
        for alpha in (0.3125, 1.0 / 3.0, -7.0):
            out = torch.full((N + PAD, Dm), SENTINEL, device=DEV)
            img = want = None
            if Dm == 128:
                nbytes = _lib.lib().call("ddfa_act_image_bytes", N)
                img = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
                want = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
            _lib_call("ddfa_stmt_scale_input", _p(x), float(alpha), N, Dm, _p(out), _p(img), _stream_ptr())
            assert torch.equal(out[:N], torch.tensor(alpha, dtype=torch.float32) * x) and bool((out[N:] == SENTINEL).all())
            if img is not None:
                _lib_call("ddfa_act_to_image", _p(out), N, Dm, _p(want), _stream_ptr())
                assert torch.equal(img, want)


# ---- DeepLiftShap / GradientShap draws ---------------------------------------------------------------------------------------
GAUSS_ULPS = 8          # device Box-Muller (logf, sqrtf, sincospif: a few ulps together) against fp64 of the same words


def _shap(x, gp, alpha, noise, base, seed, counter, sample):
    N, Dm = x.shape
    inp = torch.full((N, Dm), float("nan"), device=DEV)
    diff = torch.full((N, Dm), float("nan"), device=DEV)
    _lib_call("ddfa_stmt_shap_input", _p(x), _p(gp), gp.numel() - 1, N, Dm, float(alpha), float(noise), float(base), seed, _p(counter),
              sample, _p(inp), _p(diff), 0, _stream_ptr())
    return inp, diff


def _ulps(got, ref):
    """|got - ref| in units of the fp32 spacing at |ref| (with 2^-48 of slack for the fp64 reference near a zero of sin / cos)."""
    sp = torch.from_numpy(np.spacing(np.abs(ref.cpu().numpy()).astype(np.float32)).astype(np.float64)).to(ref.device)
    return float(((got.double() - ref).abs() / (sp + 2.0 ** -48)).max())


@pytest.mark.parametrize("Dm", R.SHAP_WIDTHS)
def test_shap_input_draws_over_3000_functions(Dm):
    """ddfa_stmt_shap_input over 3 000 functions (more than the 1 056 CTAs of its grid, empty functions among them), sample 3, a
    batch counter past 2^32 (its low word is the Philox counter word): the per-function alpha bit for bit against the host
    Philox; the two Gaussians within GAUSS_ULPS of an fp64 Box-Muller of the same words; and diff / input exactly
    fp32(x + 0.5 e) - 2 e' and fp32(alpha diff) or fp32(0.5 diff + 2 e') from the device's own Gaussians (power-of-two stdevs
    and alpha: one rounding per step, however the compiler contracts them)."""
    sizes = R.shap_sizes(Dm)
    B, N = len(sizes), int(sizes.sum())
    gp = H.graph_ptr(sizes).to(DEV)
    seed = (Dm << 40) + 12345
    counter = torch.tensor([R.SHAP_COUNTER], dtype=torch.int64, device=DEV)
    batch, sample = R.SHAP_COUNTER & 0xFFFFFFFF, 3
    x = torch.randn(N, Dm, device=DEV, generator=torch.Generator(device=DEV).manual_seed(Dm))
    zero = torch.zeros_like(x)
    gid = H.segment_ids(sizes).to(DEV)
    # the Gaussians: noise 1 on x = 0 gives diff = e; alpha = 0 and baseline 1 give input = e'
    _, e = _shap(zero, gp, 1.0, 1.0, 0.0, seed, counter, sample)
    e_b, _ = _shap(zero, gp, 0.0, 0.0, 1.0, seed, counter, sample)
    ref_e = torch.from_numpy(A.gaussians(seed, batch, sample, N, Dm, False)).to(DEV)
    ref_b = torch.from_numpy(A.gaussians(seed, batch, sample, N, Dm, True)).to(DEV)
    worst = dict(noise_ulps=_ulps(e, ref_e) / GAUSS_ULPS, baseline_ulps=_ulps(e_b, ref_b) / GAUSS_ULPS)
    # alpha drawn per function, no baseline: diff = x + 0.5 e, input = alpha_b diff
    inp, diff = _shap(x, gp, -1.0, 0.5, 0.0, seed, counter, sample)
    alpha = torch.from_numpy(A.alphas(seed, batch, sample, B)).to(DEV)[gid][:, None]
    assert torch.equal(diff, x + 0.5 * e), "diff"
    assert torch.equal(inp, alpha * diff), "alpha or input"
    # given alpha, both draws: diff = (x + 0.5 e) - 2 e', input = 0.5 diff + 2 e'
    inp, diff = _shap(x, gp, 0.5, 0.5, 2.0, seed, counter, sample)
    assert torch.equal(diff, (x + 0.5 * e) - 2 * e_b), "diff with a baseline"
    assert torch.equal(inp, 0.5 * diff + 2 * e_b), "input with a baseline"
    assert int(counter.item()) == R.SHAP_COUNTER, "the counter is read, not advanced"
    print(f"shap input D={Dm} B={B} N={N}: Gaussians within {GAUSS_ULPS * max(worst.values()):.2f} ulps")
    _report(f"stmt shap input D={Dm}", worst)


# ---- node probability ---------------------------------------------------------------------------------------------------------
def test_node_probability_row_counts():
    """ddfa_stmt_node_probability: sigmoid of the first clamp(*num_rows, 0, N) logits, zero after, for *num_rows = -1, 0, S < N,
    N and N + 5; within 8 u of float64 (expf, the add and the division), plus the subnormal rounding for logits of -100."""
    N = HUB_NODES
    logits = torch.randn(N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)) * 8
    logits[::1001], logits[5::1003] = 100.0, -100.0
    ref = torch.sigmoid(logits.double())
    worst = {}
    for nr in (-1, 0, 12_345, N, N + 5):
        S = min(max(nr, 0), N)
        scores = torch.full((N + PAD,), SENTINEL, device=DEV)
        num_rows = torch.tensor([nr], dtype=torch.int32, device=DEV)
        _lib_call("ddfa_stmt_node_probability", _p(logits), _p(num_rows), N, _p(scores), _stream_ptr())
        assert bool((scores[S:N] == 0).all()) and bool((scores[N:] == SENTINEL).all()), nr
        worst[f"rows={nr}"] = H.ratio((scores[:S].double() - ref[:S]).abs(), 8 * U * ref[:S] + 2.0 ** -126)
    _report(f"stmt node probability N={N}", worst)


# ---- the metric ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("full", [False, True])
def test_metric_edges_exactly(full):
    """ddfa_stmt_metric on statement_rule.metric_case (600 functions: more than the 264 CTAs, the last 10 as padding; a 20 000-node
    function with vulnerable ties at the top score across warps and loop iterations; the first-ranked vulnerable node in the
    last warp; +0.0 tied with -0.0; +-inf; NaN on a non-vulnerable node) against host_state, word for word, accumulated twice."""
    s, v, bnn = R.metric_case()
    num_valid = len(bnn) - 10
    n_valid = int(bnn[:num_valid].sum())
    want = R.host_state(s[:n_valid], v[:n_valid], bnn[:num_valid], full, batches=2)
    want[:R.BATCHES] *= 2
    assert want[R.NAN] == 2 and want[R.VULN] > 0
    sd, vd = torch.from_numpy(s).to(DEV), torch.from_numpy(v).to(DEV)
    gp = H.graph_ptr(bnn).to(DEV)
    st = torch.zeros(_lib.STMT_STATE_WORDS, dtype=torch.float64, device=DEV)
    ws = torch.full((_lib.lib().call("ddfa_stmt_metric_workspace_bytes"),), 0xFF, dtype=torch.uint8, device=DEV)
    mode = _lib.STMT_MODE_FULL if full else _lib.STMT_MODE_VULN_ONLY
    for _ in range(2):
        _lib_call("ddfa_stmt_metric", _p(sd), _p(vd), _p(gp), len(bnn), num_valid, mode, 0.5, _p(st), _p(ws), ws.numel(), _stream_ptr())
    got = st.cpu().numpy()
    assert np.array_equal(got, want), (got, want)
    for j, (vul, rank, _, nan) in enumerate(R.ranks(s[:int(bnn[:7].sum())], v[:int(bnn[:7].sum())], bnn[:7])):
        n0 = int(bnn[:j].sum())
        if rank is not None:
            assert rank == R.rank_by_sort(s[n0:n0 + bnn[j]], v[n0:n0 + bnn[j]]), j


# ---- statement scores on the wide tensor-core engine ------------------------------------------------------------------------
GRAD_TOL = 2e-3             # test_statements_gpu.py::GRAD_TOL["tcgen05"], relative to the largest |score|
KINK = 1e-5                 # a hidden pre-activation of the head this close to 0 in fp64 may sit on the other side in fp32


@contextlib.contextmanager
def _kink_margin(o, B):
    """Records, per function, the smallest |pre-activation| of any hidden ReLU of the oracle's head over every forward run in the
    block.  The head is piecewise linear: a unit within KINK of its kink can take the other branch in the kernels' fp32
    forward, which changes that function's input gradient by O(its weight) — a difference of the reference's branch, not of the
    kernels — so those functions are reported and left out of the comparison.  Integrated gradients run the head at inputs
    scaled down to 1 / (2 m), where many pre-activations sit near their bias and so near 0: up to a third of the functions may
    be left out there, and the error over every function is printed beside the asserted one."""
    margin = torch.full((B,), math.inf, dtype=torch.float64, device=DEV)

    def hook(mod, inp, out):
        margin.copy_(torch.minimum(margin, inp[0].detach().abs().amin(1)))
    handles = [m.register_forward_hook(hook) for m in o.output_layer if isinstance(m, torch.nn.ReLU)]
    try:
        yield margin
    finally:
        for h_ in handles:
            h_.remove()


@pytest.mark.parametrize("W", [192, 512])
def test_wide_engine_statement_scores(W):
    """FusedEvaluator(statements="saliency" / "integrated_gradients" (ig_steps = 4) / "deeplift") on the tensor-core engine at
    W = 192 and 512 (hidden W / 4, concat_all_absdf, two head layers) over the 40 001-node hub batch: the dgrad-only backward
    against the float64 oracle of tests/statement_rule.py and tests/attribution_rule.py, within GRAD_TOL x sqrt(W / 128) of the
    largest |score|; the statement state is host_state of the scores; parameters and .grad untouched."""
    hidden, steps = W // 4, 4
    g = hub_batch("mid")
    gd = g.to(DEV)
    torch.manual_seed(W)
    o = O.OracleFlowGNNGGNN("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, hidden, 4, 2, concat_all_absdf=True)
    m = D.FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, hidden, 4, 2, concat_all_absdf=True,
                            engine="tcgen05")
    m.load_state_dict(o.state_dict())
    m = m.to(DEV)
    o = o.double().to(DEV)
    assert m.engine == "tcgen05" and m._D == W
    for p in m.parameters():
        p.grad = torch.full_like(p, 0.25)
    before = [p.detach().clone() for p in m.parameters()]
    bnn = g.batch_num_nodes()
    gid = torch.repeat_interleave(torch.arange(bnn.numel()), bnn).to(DEV)
    tol = GRAD_TOL * max(1.0, (W / 128) ** 0.5)
    worst, left_out, every = {}, {}, {}
    for mode in ("saliency", "integrated_gradients", "deeplift"):
        ev = D.FusedEvaluator(m, statements=mode, ig_steps=steps)
        ev.update(g)
        torch.cuda.synchronize()
        got = ev.last_scores().clone().double()
        with _kink_margin(o, bnn.numel()) as margin:
            if mode == "saliency":
                ref = R.oracle_saliency(o, gd)
            elif mode == "integrated_gradients":
                ref = R.oracle_integrated_gradients(o, gd, steps)
            else:
                with torch.no_grad():
                    x = o.embed(gd)
                ref = A.oracle_deeplift(o, gd, [torch.zeros_like(x)])
        # DeepLift's rescale multiplier is continuous at the kink: every function is compared
        keep = (margin > KINK)[gid] if mode != "deeplift" else torch.ones_like(gid, dtype=torch.bool)
        left_out[mode] = int((margin <= KINK).sum()) if mode != "deeplift" else 0
        assert left_out[mode] <= bnn.numel() // 3, (mode, left_out[mode])
        scale = float(ref.abs().max())
        worst[mode] = float((got - ref).abs()[keep].max()) / (tol * scale)
        every[mode] = float((got - ref).abs().max()) / (tol * scale)
        st = ev.statement_state().cpu().numpy()
        assert np.array_equal(st, R.host_state(got.float().cpu().numpy(), g.ndata["_VULN"].numpy(), bnn.numpy(), False)), mode
    for p, q in zip(m.parameters(), before):
        assert torch.equal(p.detach(), q) and bool((p.grad == 0.25).all())
    _report(f"wide tc statement scores W={W} N={g.num_nodes()} (functions left out near a kink: {left_out}; over every function: "
            + ", ".join(f"{k}={v:.3g}" for k, v in every.items()) + ")", worst)
