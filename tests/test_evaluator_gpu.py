"""GPU: the evaluation metric kernels (ddfa_eval_metrics_graph / _rows) against fp64 NumPy, FusedEvaluator against the module
path (module.forward / module.validation_step) on every batch path, its independence from a FusedTrainer that trains the same
module, and FusedTrainer(track_metrics=True)."""
import math

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200 import engine as E
from deepdfa_b200.evaluator import TP, FP, TN, FN, SAMPLES, BATCHES, LOSS_W, WEIGHT, STORED, OVERFLOW

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
ENGINES = ["simt", "tcgen05"]
TINY = float(np.finfo(np.float32).tiny)     # fp32 1/(1+expf(100)) is 0, fp64 gives a denormal 3.7e-44


# ---- the kernels, through the ABI -----------------------------------------------------------------------------------------
def np_bce(x, y, pw):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    lw = 1.0 + (pw - 1.0) * y
    return (1.0 - y) * x + lw * (np.log1p(np.exp(-np.abs(x))) + np.maximum(-x, 0.0))


class Kernel:
    def __init__(self, capacity=0):
        self.state = torch.zeros(_lib.EVAL_STATE_WORDS, dtype=torch.float64, device=DEV)
        self.ws = torch.empty(_lib.lib().call("ddfa_eval_metrics_workspace_bytes"), dtype=torch.uint8, device=DEV)
        self.C = capacity
        self.probs = torch.full((max(capacity, 1),), -1.0, device=DEV) if capacity else None
        self.labels = torch.full((max(capacity, 1),), -1.0, device=DEV) if capacity else None

    def _tail(self, pw, weight):
        return (pw, weight, self.state.data_ptr(), E._p(self.probs), E._p(self.labels), self.C, self.ws.data_ptr(), self.ws.numel(),
                torch.cuda.current_stream().cuda_stream)

    def graph(self, logits, vuln, gptr, num_valid, pw, weight):
        lg, vu, gp = (torch.as_tensor(logits, dtype=torch.float32).to(DEV), torch.as_tensor(vuln, dtype=torch.int32).to(DEV),
                      torch.as_tensor(gptr, dtype=torch.int32).to(DEV))
        _lib.lib().call("ddfa_eval_metrics_graph", lg.data_ptr(), vu.data_ptr(), gp.data_ptr(), lg.numel(), num_valid,
                        *self._tail(pw, weight))
        torch.cuda.synchronize()

    def rows(self, logits, vuln, rows, S, pw, weight):
        N = len(vuln)
        lg = torch.zeros(N, dtype=torch.float32)
        lg[:len(logits)] = torch.as_tensor(logits, dtype=torch.float32)
        rw = torch.zeros(N, dtype=torch.int32)
        rw[:len(rows)] = torch.as_tensor(rows, dtype=torch.int32)
        lg, rw = lg.to(DEV), rw.to(DEV)
        vu = torch.as_tensor(vuln, dtype=torch.int32).to(DEV)
        s = torch.tensor([S], dtype=torch.int32, device=DEV)
        _lib.lib().call("ddfa_eval_metrics_rows", lg.data_ptr(), vu.data_ptr(), rw.data_ptr(), s.data_ptr(), N, *self._tail(pw, weight))
        torch.cuda.synchronize()


def expected_state(batches, pw, C=0):
    """fp64 reference state of [(logits, labels, weight)]."""
    s = np.zeros(_lib.EVAL_STATE_WORDS)
    probs = []
    for x, y, w in batches:
        x, y = np.asarray(x, np.float32), np.asarray(y, np.float64)
        p = 1.0 / (1.0 + np.exp(-x.astype(np.float64)))
        pred = p >= 0.5
        t = y != 0
        s[TP] += np.sum(pred & t); s[FP] += np.sum(pred & ~t); s[TN] += np.sum(~pred & ~t); s[FN] += np.sum(~pred & t)
        s[SAMPLES] += len(x); s[BATCHES] += 1
        if len(x):
            s[LOSS_W] += np_bce(x, y, pw).mean() * w
            s[WEIGHT] += w
        probs.extend(p.tolist())
    if C:
        s[STORED] = min(C, len(probs))
        s[OVERFLOW] = len(probs) - s[STORED]
    return s, np.asarray(probs)


def graph_case(B, seed, sizes_max=40):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, sizes_max, B)
    gptr = np.zeros(B + 1, np.int64)
    np.cumsum(sizes, out=gptr[1:])
    vuln = (rng.random(gptr[-1]) < 0.02).astype(np.int32)
    logits = rng.normal(0, 3, B).astype(np.float32)
    logits[::7] = 0.0                                   # p == 0.5 exactly: predicted positive
    logits[1::11] = 100.0
    logits[2::11] = -100.0                              # |x| = 100: the BCE stays finite
    labels = np.array([vuln[gptr[b]:gptr[b + 1]].max() for b in range(B)])
    return logits, vuln, gptr, labels


def close_state(got, want, rtol=1e-6):
    """Counts exact; the loss to fp32 precision (each term is an fp32 value, summed in fp64)."""
    got = got.cpu().numpy()
    assert np.array_equal(got[[TP, FP, TN, FN, SAMPLES, BATCHES, STORED, OVERFLOW]], want[[TP, FP, TN, FN, SAMPLES, BATCHES, STORED, OVERFLOW]])
    np.testing.assert_allclose(got[[LOSS_W, WEIGHT]], want[[LOSS_W, WEIGHT]], rtol=rtol)


def test_graph_kernel_against_fp64_with_padding_accumulation_and_reset():
    k = Kernel(capacity=12000)
    batches = []
    # 2 113 graphs and more: past the 264 CTAs x 8 warps of graph_metrics_kernel, whose warps then stride over the batch
    for i, (B, nv) in enumerate([(300, 300), (1024, 1000), (17, 12), (2112, 2112), (2113, 2100), (5000, 4990)]):
        logits, vuln, gptr, labels = graph_case(B, i)
        k.graph(logits, vuln, gptr, nv, 2.0, float(nv))
        batches.append((logits[:nv], labels[:nv], float(nv)))       # graphs [nv, B) are padding: ignored
    want, probs = expected_state(batches, 2.0, C=k.C)
    close_state(k.state, want)
    assert k.state[TP].item() + k.state[FP].item() > 0
    n = int(want[SAMPLES])
    np.testing.assert_allclose(k.probs[:n].cpu().numpy(), probs, rtol=2e-7, atol=TINY)
    assert np.array_equal(k.labels[:n].cpu().numpy(), np.concatenate([b[1] for b in batches]).astype(np.float32))
    assert float(k.probs[n].item()) == -1.0, "nothing written past the samples"
    k.state.zero_()
    logits, vuln, gptr, labels = graph_case(50, 9)
    k.graph(logits, vuln, gptr, 50, 1.0, 50.0)
    want, _ = expected_state([(logits, labels, 50.0)], 1.0, C=k.C)
    close_state(k.state, want)


def test_zero_and_large_logits():
    k = Kernel()
    k.graph([0.0, 0.0, 100.0, -100.0, 100.0, -100.0], [0, 1, 0, 1, 1, 0], list(range(7)), 6, 2.0, 6.0)
    s = k.state.cpu().numpy()
    # x = 0 -> positive; 100 on a negative is FP, -100 on a positive is FN
    assert (s[TP], s[FP], s[TN], s[FN]) == (2, 2, 1, 1)
    terms = [math.log(2), 2 * math.log(2), 100.0, 200.0, 0.0, 0.0]
    assert math.isfinite(s[LOSS_W]) and abs(s[LOSS_W] - np.mean(terms) * 6) < 1e-5


def test_row_kernel_against_fp64():
    rng = np.random.default_rng(3)
    N = 40000
    vuln = (rng.random(N) < 0.1).astype(np.int32)
    k = Kernel(capacity=100000)
    batches = []
    for S in (31000, 0, 17):
        rows = np.sort(rng.choice(N - 100, S, replace=False)).astype(np.int32)
        logits = rng.normal(0, 2, S).astype(np.float32)
        if S:
            logits[::13] = 0.0
        k.rows(logits, vuln, rows, S, 2.0, 64.0)
        batches.append((logits, vuln[rows], 64.0))
    want, probs = expected_state(batches, 2.0, C=100000)
    close_state(k.state, want)
    assert k.state[BATCHES].item() == 3 and k.state[WEIGHT].item() == 128.0, "the empty batch adds no loss weight"
    np.testing.assert_allclose(k.probs[:len(probs)].cpu().numpy(), probs, rtol=2e-7, atol=TINY)


def test_prediction_overflow_keeps_counts_complete():
    k = Kernel(capacity=100)
    batches = []
    for i in range(3):
        logits, vuln, gptr, labels = graph_case(60, 20 + i)
        k.graph(logits, vuln, gptr, 60, 1.0, 60.0)
        batches.append((logits, labels, 60.0))
    want, probs = expected_state(batches, 1.0, C=100)
    close_state(k.state, want)
    assert k.state[STORED].item() == 100 and k.state[OVERFLOW].item() == 80
    np.testing.assert_allclose(k.probs[:100].cpu().numpy(), probs[:100], rtol=2e-7, atol=TINY)


@pytest.mark.parametrize("det", ["0", "1"])
def test_state_is_bit_reproducible(det, monkeypatch):
    monkeypatch.setenv("DDFA_DETERMINISTIC", det)
    _lib.apply_deterministic_mode()
    states = []
    for _ in range(2):
        k = Kernel(capacity=10)
        for i in range(4):
            logits, vuln, gptr, _ = graph_case(2000, 40 + i)
            k.graph(logits, vuln, gptr, 1990, 2.0, 1990.0)
        states.append(k.state.cpu())
    assert torch.equal(states[0], states[1])


# ---- against the module path ----------------------------------------------------------------------------------------------
def make_module(engine, style, seed=0, **kw):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine, label_style=style,
                               **kw).to(DEV)


def batch_list(style, seed=0):
    rate = 0.004 if style == "graph" else 0.1
    return [synth.make_batch(n, 30, seed=seed + i, variable=True, vuln_rate=rate) for i, n in enumerate((17, 64, 255, 40))]


def module_reference(m, batches):
    """(probs, labels, loss) of module.validation_step over the batches: probs / labels concatenated, the Lightning epoch loss."""
    probs, labels, lw, w = [], [], 0.0, 0.0
    for b in batches:
        loss, p, y = m.validation_step((b.to(DEV), {}))
        probs.append(p.float())
        labels.append(y)
        lw += float(loss) * b.batch_size
        w += b.batch_size
    return torch.cat(probs), torch.cat(labels), lw / w


def counts(probs, labels):
    pred, t = probs >= 0.5, labels != 0
    return [int((pred & t).sum()), int((pred & ~t).sum()), int((~pred & ~t).sum()), int((~pred & t).sum())]


def ulps(a, b):
    ai = a.contiguous().view(torch.int32).long()
    bi = b.contiguous().view(torch.int32).long()
    return int((ai - bi).abs().max()) if a.numel() else 0


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("style", ["graph", "node"])
def test_against_module_path(engine, style):
    m = make_module(engine, style)
    batches = batch_list(style)
    ref_p, ref_y, ref_loss = module_reference(m, batches)
    ev = D.FusedEvaluator(m, use_cuda_graph=True, max_predictions=ref_p.numel())
    for b in batches:
        ev.update(b)
    res = ev.compute("val_")
    probs, labels = ev.predictions()
    dev_ulp = ulps(probs, ref_p)
    print(f"{engine}/{style}: {probs.numel()} samples, max deviation from torch.sigmoid(module.forward) = {dev_ulp} ulp")
    assert probs.numel() == ref_p.numel()
    # graph style runs the module's readout + MLP kernel: measured 0 ulp on H100.  Node style runs the row-list head
    # (ddfa_node_head_fwd) where the module runs the readout over one-node graphs: the same products summed in another
    # order, measured 4 ulp (both engines) on H100.
    assert dev_ulp <= (1 if style == "graph" else 8)
    assert torch.equal(labels, ref_y.float())
    tn, fp = res["val_confusion"][0]
    fn, tp = res["val_confusion"][1]
    assert [tp, fp, tn, fn] == counts(ref_p, ref_y)
    assert abs(res["val_loss"] - ref_loss) <= 1e-6 * abs(ref_loss)

    # bucketing: one padding graph per batch (255 -> 256 graphs can switch the readout's MLP path): close, same decisions
    evb = D.FusedEvaluator(m, use_cuda_graph=True, bucket_nodes=512, bucket_edges=1024, max_predictions=ref_p.numel())
    for b in batches:
        evb.update(b)
    rb = evb.compute("val_")
    pb, _ = evb.predictions()
    assert (pb - ref_p).abs().max().item() <= 1e-6
    assert torch.equal(pb >= 0.5, ref_p >= 0.5)
    assert rb["val_confusion"] == res["val_confusion"]
    assert abs(rb["val_loss"] - ref_loss) <= 1e-6 * abs(ref_loss)


@pytest.mark.parametrize("style", ["graph", "node"])
def test_paths_give_the_same_state(style):
    m = make_module("tcgen05", style)
    batches = batch_list(style, seed=10)
    arena = D.GraphArena.from_graphs(batches, device=DEV)
    offs = np.cumsum([0] + [b.batch_size for b in batches])
    dev_batches = [b.to(DEV) for b in batches]

    def run(fn, ev, passes=3):
        for _ in range(passes):
            for i, b in enumerate(batches):
                fn(ev, i, b)
        return ev.state().clone()

    host = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m))
    eager = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, use_cuda_graph=False))
    res_ev = D.FusedEvaluator(m)
    resident = run(lambda ev, i, b: ev.update(dev_batches[i]), res_ev)
    assert len(res_ev._graphs) == len(batches), "one captured graph per resident batch"
    ids = run(lambda ev, i, b: ev.update_ids(arena, np.arange(offs[i], offs[i + 1])), D.FusedEvaluator(m))

    def prefetched(ev, i, b):
        if i + 1 < len(batches):
            ev.prefetch(batches[i + 1])
        ev.update(b)
    pre = run(prefetched, D.FusedEvaluator(m))
    few = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, max_graph_shapes=1))     # eager beyond the first shape
    for name, s in (("eager", eager), ("resident", resident), ("ids", ids), ("prefetch", pre), ("max_graph_shapes=1", few)):
        assert torch.equal(s, host), name
    bucketed = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, bucket_nodes=512, bucket_edges=1024))
    bucketed_eager = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, use_cuda_graph=False, bucket_nodes=512))
    for s in (bucketed, bucketed_eager):
        assert torch.equal(s[[TP, FP, TN, FN, SAMPLES, BATCHES, WEIGHT]], host[[TP, FP, TN, FN, SAMPLES, BATCHES, WEIGHT]])
        assert abs(float(s[LOSS_W] - host[LOSS_W])) <= 1e-6 * abs(float(host[LOSS_W]))


@pytest.mark.parametrize("style", ["graph", "node"])
def test_exact_boundary_when_the_last_layer_is_zero(style):
    m = make_module("simt", style)
    with torch.no_grad():
        m.output_layer[-1].weight.zero_()
        m.output_layer[-1].bias.zero_()
    batches = batch_list(style, seed=20)
    ev = D.FusedEvaluator(m)
    lw = w = 0.0
    for b in batches:
        ev.update(b)
        y = m.get_label(b.to(DEV)).cpu().double()
        lw += float((y * 2.0 * math.log(2) + (1 - y) * math.log(2)).mean()) * b.batch_size
        w += b.batch_size
    r = ev.compute("test_")
    assert r["test_confusion"][0][0] == 0 and r["test_confusion"][1][0] == 0, "every sample predicted positive"
    assert r["test_Recall"] == 1.0
    assert abs(r["test_loss"] - lw / w) <= 1e-6 * (lw / w)


def test_compute_raises_on_empty_overflow_and_bad_indices():
    m = make_module("simt", "graph")
    ev = D.FusedEvaluator(m, max_predictions=10)
    with pytest.raises(ValueError, match="no sample"):
        ev.compute()
    ev.update(synth.make_batch(16, 20, seed=1))
    with pytest.raises(ValueError, match="max_predictions >= 16"):
        ev.compute()
    b = synth.make_batch(8, 20, seed=2)
    b.ndata[next(k for k in b.ndata if k != "_VULN")][3] = 5000
    ev2 = D.FusedEvaluator(m)
    ev2.update(b)
    with pytest.raises(IndexError):
        ev2.compute()


@pytest.mark.parametrize("style", ["graph", "node"])
def test_c1_batch(style):
    m = make_module("tcgen05", style)
    b = synth.make_batch(1024, 150, seed=0, variable=True, vuln_rate=0.0004 if style == "graph" else 0.06)
    ev = D.FusedEvaluator(m)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ev.update(b)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"C1 {style}: {b.num_nodes()} nodes, first-batch peak allocation {peak / 2 ** 20:.1f} MiB")
    assert peak < 2 ** 30
    r = ev.compute()
    p, y, _ = module_reference(m, [b])
    assert [r["val_confusion"][1][1], r["val_confusion"][0][1], r["val_confusion"][0][0], r["val_confusion"][1][0]] == counts(p, y)
    assert r["val_num_samples"] == (1024 if style == "graph" else b.num_nodes())


# ---- alongside a FusedTrainer ---------------------------------------------------------------------------------------------
def test_evaluation_does_not_change_training(monkeypatch):
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
    train = [synth.make_batch(32, 30, seed=100 + i, variable=True, vuln_rate=0.01) for i in range(4)]
    val = batch_list("graph", seed=50)

    def run(with_eval):
        m = make_module("tcgen05", "graph", seed=3)
        early = D.FusedEvaluator(m)
        if with_eval:
            for _ in range(3):                      # captured over the module's own parameter storage
                early.reset()
                for b in val:
                    early.update(b)
        tr = D.FusedTrainer(m, use_cuda_graph=True, distributed=False)
        ev = D.FusedEvaluator(m)
        losses = []
        for b in train:
            losses.append(float(tr.step(b)))
            if with_eval:
                ev.reset()
                for v in val:
                    ev.update(v)
                ev.compute()
        states = []
        for e in (early, D.FusedEvaluator(m)):
            e.reset()
            for v in val:
                e.update(v)
            states.append(e.state().clone())
        return losses, tr.flat_p.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone(), states

    a, b = run(False), run(True)
    assert a[0] == b[0]
    for x, y in zip(a[1:4], b[1:4]):
        assert torch.equal(x, y)
    assert torch.equal(b[4][0], b[4][1]), "an evaluator built before the trainer evaluates the trained weights"


def test_track_metrics_graph_style():
    m = make_module("tcgen05", "graph", seed=4)
    tr = D.FusedTrainer(m, track_metrics=True, distributed=False)
    want, near = np.zeros(4), 0
    for i in range(4):
        b = synth.make_batch(48, 30, seed=200 + i, variable=True, vuln_rate=0.01)
        with torch.no_grad():
            p = torch.sigmoid(m(b.to(DEV), {}))
        y = m.get_label(b.to(DEV))
        want += counts(p, y)
        near += int(((p - 0.5).abs() < 1e-6).sum())
        tr.step(b)
    r = tr.metrics("train_")
    got = [r["train_confusion"][1][1], r["train_confusion"][0][1], r["train_confusion"][0][0], r["train_confusion"][1][0]]
    assert np.abs(np.asarray(got) - want).sum() <= 2 * near
    assert r["train_num_samples"] == 4 * 48 and math.isfinite(r["train_loss"])
    tr.reset_metrics()
    with pytest.raises(ValueError):
        tr.metrics()


def test_track_metrics_node_style_counts_the_loss_rows():
    m = make_module("simt", "node", seed=5, undersample_node_on_loss_factor=1.0)
    tr = D.FusedTrainer(m, track_metrics=True, distributed=False)
    n_rows = 0
    for i in range(3):
        b = synth.make_batch(24, 30, seed=300 + i, variable=True, vuln_rate=0.1)
        tr.step(b)
        n_rows += tr.last_loss_rows().numel()
    assert tr.metrics()["train_num_samples"] == n_rows


@pytest.mark.parametrize("style", ["graph", "node"])
def test_track_metrics_adds_exactly_the_metric_launches(style):
    b = synth.make_batch(24, 30, seed=7, variable=True, vuln_rate=0.05).to(DEV)
    launches = {}
    for track in (False, True):
        m = make_module("simt", style, seed=6)
        tr = D.FusedTrainer(m, track_metrics=track, distributed=False)
        tr.step(b)
        torch.cuda.synchronize()
        l0 = _lib.lib().call("ddfa_launch_count")
        tr.step(b)
        torch.cuda.synchronize()
        launches[track] = _lib.lib().call("ddfa_launch_count") - l0
    assert launches[True] - launches[False] == 2       # the metric kernel and its one-thread finish
