"""GPU: statement-level localisation in FusedEvaluator (statements=...).  ddfa_stmt_metric against the host restatement of its
ranking rule (tests/statement_rule.py), exactly, on constructed ties across warp and CTA boundaries, hub-sized functions, padding
and the reference golden; the per-node scores (attention, saliency, integrated gradients, probability) against the fp64 oracle
with torch.autograd; host, resident, arena and prefetched paths bit-identical (bucketed: captured equals eager); deterministic repeats; parameters, .grad and a FusedTrainer untouched; and
the launch count of statements=None unchanged."""
import os
import sys

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from oracle import ggnn_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import statement_rule as R  # noqa: E402
from test_statements_cpu import GOLDEN, IG_COMPLETENESS_BOUND  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
GRAD_TOL = {"simt": 2e-4, "tcgen05": 2e-3}     # relative to the largest entry: tests/test_parity_gpu.py's module-gradient bounds


def c0(seed=0, rate=0.3):
    return synth.make_batch(256, 150, seed=seed, variable=True, vuln_rate=rate)


def c1(seed=0, rate=0.3):
    return synth.make_batch(1024, 150, seed=seed, variable=True, vuln_rate=rate)


# ---- the metric kernel, through the ABI ------------------------------------------------------------------------------------
def kernel_state(scores, vuln, bnn, num_valid, full, states=None):
    s = torch.as_tensor(np.asarray(scores, np.float32)).to(DEV)
    v = torch.as_tensor(np.asarray(vuln, np.int32)).to(DEV)
    gp = torch.as_tensor(np.concatenate([[0], np.cumsum(bnn)]).astype(np.int32)).to(DEV)
    st = torch.zeros(_lib.STMT_STATE_WORDS, dtype=torch.float64, device=DEV) if states is None else states
    ws = torch.empty(_lib.lib().call("ddfa_stmt_metric_workspace_bytes"), dtype=torch.uint8, device=DEV)
    _lib.lib().call("ddfa_stmt_metric", s.data_ptr(), v.data_ptr(), gp.data_ptr(), len(bnn), num_valid,
                    _lib.STMT_MODE_FULL if full else _lib.STMT_MODE_VULN_ONLY, 0.5, st.data_ptr(), ws.data_ptr(), ws.numel(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return st.cpu().numpy()


def constructed_case(seed):
    """Functions whose sizes straddle the warp (32) and CTA (128) widths up to hub size, scores on a grid of 4 values (ties
    everywhere), the first-ranked vulnerable node placed just after a warp / CTA boundary behind an equal non-vulnerable score."""
    rng = np.random.default_rng(seed)
    sizes = [1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 3001, 9000] + list(rng.integers(1, 60, size=300))
    scores, vuln = [], []
    for n in sizes:
        s = (rng.integers(0, 4, size=n) / 4).astype(np.float32)
        v = (rng.random(n) < 0.05).astype(np.int32)
        if n > 130 and rng.random() < 0.8:
            s[:] = np.minimum(s, np.float32(0.5))
            v[:] = 0
            for j in (32, 128, min(n - 1, 129)):       # equal top scores across boundaries: only the lowest vulnerable id counts
                s[j] = 0.75
            v[min(n - 1, 129)] = 1
            v[128] = rng.integers(0, 2)
        scores.append(s)
        vuln.append(v)
    return np.concatenate(scores), np.concatenate(vuln), np.array(sizes)


@pytest.mark.parametrize("full", [False, True])
def test_metric_kernel_matches_the_host_rule(full):
    for seed in range(3):
        s, v, bnn = constructed_case(seed)
        for nv in (len(bnn), len(bnn) - 7):           # the last graphs as bucket padding
            got = kernel_state(s, v, bnn[:len(bnn)], nv, full)
            n_nodes = int(bnn[:nv].sum())
            want = R.host_state(s[:n_nodes], v[:n_nodes], bnn[:nv], full)
            assert np.array_equal(got, want), (seed, nv, got, want)
    for case in torch.load(GOLDEN)["cases"]:
        bnn = case["batch_num_nodes"].numpy()
        got = kernel_state(case["scores"].numpy(), case["vuln"].numpy(), bnn, len(bnn), full)
        assert np.array_equal(got, R.host_state(case["scores"].numpy(), case["vuln"].numpy(), bnn, full)), case["name"]
        if full:
            m = D.FusedEvaluator.statement_metrics_from_state(got, "t_", node_style=True)
            for k in range(1, 11):
                if case["vo"] is not None:
                    assert m[f"t_stmt_top{k}"] == case["vo"][k]
                if case["all"] is not None:
                    assert m[f"t_stmt_all_top{k}"] == case["all"][k]


def test_metric_kernel_counts_nan_and_accumulates():
    s, v, bnn = constructed_case(7)
    s = s.copy()
    s[5] = np.nan
    st = torch.zeros(_lib.STMT_STATE_WORDS, dtype=torch.float64, device=DEV)
    kernel_state(s, v, bnn, len(bnn), True, st)
    got = kernel_state(s, v, bnn, len(bnn), True, st)
    want = R.host_state(s, v, bnn, True, batches=2)
    want[:15] *= 2
    assert np.array_equal(got, want) and got[R.NAN] == 2


# ---- the scores against the fp64 oracle -------------------------------------------------------------------------------------
def make_pair(engine, hidden, style="graph", seed=0):
    torch.manual_seed(seed)
    o = O.OracleFlowGNNGGNN(FEAT, 1002, hidden, 4, 2, concat_all_absdf=True, label_style=style)
    m = D.FlowGNNGGNNModule(FEAT, 1002, hidden, 4, 2, concat_all_absdf=True, engine=engine, label_style=style)
    m.load_state_dict(o.state_dict())
    return m.to(DEV), o.double()


def scores_of(ev, b):
    ev.update(b)
    torch.cuda.synchronize()
    return ev.last_scores().clone()


ENGINE_WIDTHS = [("simt", 20), ("simt", 32), ("tcgen05", 32)]      # hidden 20: D = 80 (SIMT only); hidden 32: D = 128


@pytest.mark.parametrize("engine,hidden", ENGINE_WIDTHS)
def test_scores_match_the_oracle(engine, hidden):
    m, o = make_pair(engine, hidden)
    b = c0(seed=1)
    bnn = b.batch_num_nodes()
    gid = torch.repeat_interleave(torch.arange(bnn.numel()), bnn)
    vuln = b.ndata["_VULN"].numpy()
    for mode in ("attention", "saliency", "integrated_gradients"):
        steps = 8
        ev = D.FusedEvaluator(m, statements=mode, ig_steps=steps)
        got = scores_of(ev, b).cpu().double()
        assert got.numel() == b.num_nodes()
        if mode == "attention":
            ref = R.oracle_attention(o, b)
            err = float((got - ref).abs().max())
            sums = torch.zeros(bnn.numel(), dtype=torch.float64).index_add_(0, gid, got)
            assert err <= 1e-5 and float((sums - 1).abs().max()) <= 1e-5, (err, sums)
        else:
            ref = R.oracle_saliency(o, b) if mode == "saliency" else R.oracle_integrated_gradients(o, b, steps)
            err = float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
            assert err <= GRAD_TOL[engine], (mode, err)
        print(f"{engine}/W={4 * hidden} {mode}: max deviation {err:.2e}")
        st = ev.statement_state().cpu().numpy()
        assert np.array_equal(st, R.host_state(got.float().numpy(), vuln, bnn.numpy(), False)), mode
        r = ev.compute("test_")
        assert r["test_stmt_functions"] == 256 and "test_stmt_all_top1" not in r


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_integrated_gradients_completeness(engine):
    m, o = make_pair(engine, 32, seed=2)
    b = c0(seed=3)
    bnn = b.batch_num_nodes()
    gid = torch.repeat_interleave(torch.arange(bnn.numel()), bnn)
    with torch.no_grad():
        x = o.embed(b)
        delta = R.oracle_logits_from_x(o, b, x) - R.oracle_logits_from_x(o, b, torch.zeros_like(x))
    scale = max(float(delta.abs().max()), 1.0)
    for steps in (16, 50):
        got = scores_of(D.FusedEvaluator(m, statements="integrated_gradients", ig_steps=steps), b).cpu().double()
        sums = torch.zeros(bnn.numel(), dtype=torch.float64).index_add_(0, gid, got)
        err = float((sums - delta).abs().max())
        print(f"{engine} IG m={steps}: completeness error {err:.2e} (|delta| up to {scale:.2e})")
        assert err <= (IG_COMPLETENESS_BOUND[steps] + GRAD_TOL[engine]) * scale


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_node_probability_and_metric(engine):
    m, _ = make_pair(engine, 32, style="node", seed=4)
    b = c0(seed=5, rate=0.06)
    ev = D.FusedEvaluator(m, statements="probability", max_predictions=b.num_nodes())
    got = scores_of(ev, b)
    probs, _ = ev.predictions()
    assert torch.equal(got, probs)
    bnn = b.batch_num_nodes().numpy()
    assert np.array_equal(ev.statement_state().cpu().numpy(), R.host_state(got.cpu().numpy(), b.ndata["_VULN"].numpy(), bnn, True))
    r = ev.compute("test_")
    assert r["test_stmt_all_top10"] == r["test_stmt_top10"] * r["test_stmt_nonvuln_clean"]


# ---- batch paths, capture, determinism, side effects ------------------------------------------------------------------------
MODES = [("graph", "attention"), ("graph", "saliency"), ("graph", "integrated_gradients"), ("node", "probability")]


@pytest.mark.parametrize("style,mode", MODES)
def test_paths_give_bit_identical_scores_and_state(style, mode):
    m, _ = make_pair("tcgen05", 32, style=style, seed=6)
    rate = 0.3 if style == "graph" else 0.06
    batches = [synth.make_batch(n, 60, seed=10 + i, variable=True, vuln_rate=rate) for i, n in enumerate((17, 64, 255))]
    arena = D.GraphArena.from_graphs(batches, device=DEV)
    offs = np.cumsum([0] + [b.batch_size for b in batches])
    dev_batches = [b.to(DEV) for b in batches]

    def run(fn, ev, passes=3):
        out = []
        for _ in range(passes):
            for i, b in enumerate(batches):
                fn(ev, i, b)
                torch.cuda.synchronize()
                out.append(ev.last_scores().clone())
        return out, ev.statement_state().clone()

    kw = dict(statements=mode, ig_steps=4)
    host = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, **kw))
    eager = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, use_cuda_graph=False, **kw))
    resident = run(lambda ev, i, b: ev.update(dev_batches[i]), D.FusedEvaluator(m, **kw))
    ids = run(lambda ev, i, b: ev.update_ids(arena, np.arange(offs[i], offs[i + 1])), D.FusedEvaluator(m, **kw))

    def prefetched(ev, i, b):
        if i + 1 < len(batches):
            ev.prefetch(batches[i + 1])
        ev.update(b)
    pre = run(prefetched, D.FusedEvaluator(m, **kw))
    for name, (sc, st) in (("eager", eager), ("resident", resident), ("ids", ids), ("prefetch", pre)):
        assert torch.equal(st, host[1]), name
        for a, b in zip(sc, host[0]):
            assert torch.equal(a, b), name
    assert host[1][R.BATCHES] == 9
    # bucketing adds a padding graph (255 -> 256 graphs can switch the readout's MLP path, as in test_evaluator_gpu.py): captured
    # and eager agree bit for bit, the padding graph's nodes are left out, and the scores stay close to the unpadded ones
    bkw = dict(bucket_nodes=512, bucket_edges=1024, **kw)
    bucketed = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, **bkw))
    bucketed_eager = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, use_cuda_graph=False, **bkw))
    assert torch.equal(bucketed[1], bucketed_eager[1])
    for a, b, h in zip(bucketed[0], bucketed_eager[0], host[0]):
        assert torch.equal(a, b) and a.shape == h.shape
        assert float((a - h).abs().max()) <= 1e-4 * max(float(h.abs().max()), 1e-30)
    want = np.zeros(R.WORDS)
    for i, b in enumerate(batches * 3):
        want += R.host_state(bucketed[0][i].cpu().numpy(), b.ndata["_VULN"].numpy(), b.batch_num_nodes().numpy(), style == "node")
    assert np.array_equal(bucketed[1].cpu().numpy(), want)


@pytest.mark.parametrize("mode", ["saliency", "integrated_gradients"])
def test_deterministic_repeats_and_nothing_is_written(mode, monkeypatch):
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
    m, _ = make_pair("tcgen05", 32, seed=8)
    b = c1(seed=9)
    for p in m.parameters():
        p.grad = torch.full_like(p, 0.25)
    before = [p.detach().clone() for p in m.parameters()]
    runs = []
    for _ in range(2):
        ev = D.FusedEvaluator(m, statements=mode, ig_steps=4)
        runs.append((scores_of(ev, b), ev.statement_state().clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    for p, q in zip(m.parameters(), before):
        assert torch.equal(p.detach(), q) and bool((p.grad == 0.25).all())


def test_plain_evaluator_launch_count_is_unchanged():
    m, _ = make_pair("tcgen05", 32, seed=10)
    b = c0(seed=11)
    L = _lib.lib()
    counts = []
    for kw in ({}, dict(statements=None, ig_steps=50)):
        ev = D.FusedEvaluator(m, use_cuda_graph=False, **kw)
        ev.update(b)
        torch.cuda.synchronize()
        l0 = L.call("ddfa_launch_count")
        ev.update(b)
        torch.cuda.synchronize()
        counts.append(L.call("ddfa_launch_count") - l0)
    # the eager launch count of today's evaluator batch: the inference forward (embedding, fold, prepare, T gathers + steps,
    # readout) and the two metric launches
    assert counts[0] == counts[1]
    ev = D.FusedEvaluator(m, use_cuda_graph=False, statements="attention")
    ev.update(b)
    torch.cuda.synchronize()
    l0 = L.call("ddfa_launch_count")
    ev.update(b)
    torch.cuda.synchronize()
    assert L.call("ddfa_launch_count") - l0 == counts[0] + 3        # alpha + the statement metric's two launches


def test_evaluation_does_not_change_training(monkeypatch):
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
    train = [synth.make_batch(32, 30, seed=100 + i, variable=True, vuln_rate=0.01) for i in range(3)]
    val = [synth.make_batch(n, 30, seed=50 + i, variable=True, vuln_rate=0.3) for i, n in enumerate((17, 64))]

    def run(with_eval):
        m, _ = make_pair("tcgen05", 32, seed=3)
        tr = D.FusedTrainer(m, use_cuda_graph=True, distributed=False)
        ev = D.FusedEvaluator(m, statements="integrated_gradients", ig_steps=3)
        losses = []
        for b in train:
            losses.append(float(tr.step(b)))
            if with_eval:
                ev.reset()
                for v in val:
                    ev.update(v)
                ev.compute()
        return losses, tr.flat_p.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone()

    a, b = run(False), run(True)
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        assert torch.equal(x, y)


def test_constructor_errors():
    g, _ = make_pair("simt", 32)
    n, _ = make_pair("simt", 32, style="node")
    with pytest.raises(ValueError, match="label_style"):
        D.FusedEvaluator(g, statements="probability")
    with pytest.raises(ValueError, match="label_style"):
        D.FusedEvaluator(n, statements="saliency")
    with pytest.raises(ValueError, match="ig_steps"):
        D.FusedEvaluator(g, statements="integrated_gradients", ig_steps=0)
    with pytest.raises(ValueError, match="not one of"):
        D.FusedEvaluator(g, statements="gradcam")
    torch.manual_seed(0)
    enc = D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, concat_all_absdf=True, encoder_mode=True).to(DEV)
    with pytest.raises(ValueError, match="encoder_mode"):
        D.FusedEvaluator(enc, statements="attention")
    with pytest.raises(ValueError, match="statements=None"):
        D.FusedEvaluator(g).last_scores()
    ev = D.FusedEvaluator(g, statements="saliency")
    b = synth.make_batch(8, 20, seed=1, vuln_rate=0.5)
    ev.update(b)
    ev.statement_state()[R.NAN] = 1.0
    with pytest.raises(ValueError, match="NaN"):
        ev.compute()
    ev.reset()
    assert float(ev.statement_state().abs().sum()) == 0.0
