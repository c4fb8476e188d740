"""GPU: ddfa_predict_store through the C ABI against the host ranking (tests/predict_rule.py), and FusedPredictor against the
module and FusedEvaluator on every module kind, statement mode and batch path."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import predict_rule as R  # noqa: E402

import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200 import engine as E  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


# ---- the kernel, through the ABI ------------------------------------------------------------------------------------------
class Store:
    """A result store of ``capacity`` functions and its cursor, filled by ddfa_predict_store calls."""

    def __init__(self, capacity, k, out_dim=0, prob=False):
        self.C, self.k = capacity, k
        c = max(capacity, 1)
        self.cursor = torch.zeros(2, dtype=torch.int64, device=DEV)
        self.prob = torch.full((c,), -7.0, device=DEV) if prob else None
        self.emb = torch.full((c, out_dim), -7.0, device=DEV) if out_dim else None
        self.idx = torch.full((c, k), -7, dtype=torch.int32, device=DEV) if k else None
        self.score = torch.full((c, k), -7.0, device=DEV) if k else None

    def call(self, scores, bnn, num_valid=None, logits=None, node_probs=None, pooled=None):
        bnn = np.asarray(bnn, np.int64)
        B = len(bnn)
        gptr = torch.from_numpy(np.concatenate([[0], np.cumsum(bnn)]).astype(np.int32)).to(DEV)
        sc = torch.from_numpy(np.asarray(scores, np.float32)).to(DEV) if self.k else None
        lg = torch.from_numpy(np.asarray(logits, np.float32)).to(DEV) if logits is not None else None
        npb = torch.from_numpy(np.asarray(node_probs, np.float32)).to(DEV) if node_probs is not None else None
        pl = torch.from_numpy(np.asarray(pooled, np.float32)).to(DEV) if pooled is not None else None
        _lib.lib().call("ddfa_predict_store", E._p(lg), E._p(npb), E._p(pl), 0 if pl is None else pl.shape[1], E._p(sc), self.k,
                        gptr.data_ptr(), B, B if num_valid is None else num_valid, E._p(self.prob), E._p(self.emb), E._p(self.idx),
                        E._p(self.score), self.cursor.data_ptr(), self.C, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()


def segments(lengths, seed):
    """Scores of functions of the given lengths on a 5-value grid (ties everywhere) with -0.0, +-inf and NaN sprinkled in."""
    rng = np.random.default_rng(seed)
    n = int(np.sum(lengths))
    s = (rng.integers(0, 5, n) / 4).astype(np.float32)
    special = np.array([-0.0, np.inf, -np.inf, np.nan], np.float32)
    pick = rng.random(n) < 0.05
    s[pick] = rng.choice(special, int(pick.sum()))
    return s


def check_topk(store, scores, bnn, first=0):
    want_i, want_s = R.store(scores, bnn, store.k)
    F = len(want_i)
    got_i = store.idx[first:first + F].cpu().numpy()
    got_s = store.score[first:first + F].cpu().numpy()
    assert np.array_equal(got_i, want_i)
    assert R.same_floats(got_s, want_s)
    # the stored score is the raw score of the stored node, bit for bit (-0.0 and NaN payloads included)
    n0 = np.concatenate([[0], np.cumsum(bnn)])[:-1]
    ok = got_i >= 0
    rows = (n0[:, None] + np.maximum(got_i, 0))[ok]
    assert R.same_bits(got_s[ok], np.asarray(scores, np.float32)[rows])


@pytest.mark.parametrize("k", [1, 10, 32])
def test_segment_lengths_against_the_host_ranking(k):
    lengths = [0, 1, max(k - 1, 0), k, k + 1, 150, 5000, 100_000, 0, 3]
    s = segments(lengths, k)
    st = Store(len(lengths), k)
    st.call(s, lengths)
    check_topk(st, s, lengths)
    assert st.cursor.tolist() == [len(lengths), 0]


@pytest.mark.parametrize("k", [1, 10, 32])
def test_all_equal_infinities_and_nan(k):
    fns = [np.full(70, 0.25, np.float32), np.full(40, np.inf, np.float32), np.full(40, -np.inf, np.float32),
           np.full(33, np.nan, np.float32), np.array([np.nan, -np.inf, 1.0, np.inf, np.nan, -0.0, 0.0, -np.inf], np.float32),
           np.where(np.arange(300) % 2 == 0, np.float32(-0.0), np.float32(0.0)).astype(np.float32)]
    s = np.concatenate(fns)
    st = Store(len(fns), k)
    st.call(s, [len(f) for f in fns])
    check_topk(st, s, [len(f) for f in fns])


def test_4096_functions_padding_probabilities_and_embeddings():
    rng = np.random.default_rng(5)
    bnn = rng.integers(0, 60, 4096)
    s = segments(bnn, 11)
    logits = rng.normal(0, 4, 4096).astype(np.float32)
    logits[::97] = np.nan
    pooled = rng.normal(0, 1, (4096, 12)).astype(np.float32)
    st = Store(5000, 10, out_dim=12, prob=True)
    st.call(s, bnn, num_valid=4000, logits=logits, pooled=pooled)        # functions [4000, 4096) are padding
    assert st.cursor.tolist() == [4000, 0]
    check_topk(st, s[:int(bnn[:4000].sum())], bnn[:4000])
    lt = torch.from_numpy(logits[:4000]).to(DEV)
    assert R.same_floats(st.prob[:4000].cpu().numpy(), (1.0 / (1.0 + torch.exp(-lt))).cpu().numpy())
    assert R.same_bits(st.emb[:4000].cpu().numpy(), pooled[:4000])
    assert (st.prob[4000:].cpu() == -7.0).all() and (st.idx[4000:].cpu() == -7).all(), "nothing written past the valid functions"


def test_node_probabilities_take_the_maximum_and_pass_nan():
    rng = np.random.default_rng(6)
    bnn = np.array([5, 0, 1, 300, 7, 129])
    p = rng.random(int(bnn.sum())).astype(np.float32)
    p[6 + 200] = np.nan                               # in the 300-node function
    st = Store(10, 0, prob=True)
    st.call(None, bnn, node_probs=p)
    n0 = np.concatenate([[0], np.cumsum(bnn)])
    want = [0.0 if n == 0 else (np.nan if np.isnan(p[a:a + n]).any() else p[a:a + n].max()) for a, n in zip(n0, bnn)]
    assert R.same_floats(st.prob[:6].cpu().numpy(), np.asarray(want, np.float32))


def test_capacity_runs_out_mid_batch_and_calls_append():
    bnn1, bnn2, bnn3 = [3, 12, 0, 40, 9], [1, 20, 7], [4, 4]
    s1, s2, s3 = segments(bnn1, 1), segments(bnn2, 2), segments(bnn3, 3)
    st = Store(7, 5)
    st.call(s1, bnn1)
    assert st.cursor.tolist() == [5, 0]
    st.call(s2, bnn2)                                   # two more fit, the third is dropped
    assert st.cursor.tolist() == [7, 1]
    check_topk(st, s1, bnn1, first=0)
    check_topk(st, s2[:21], bnn2[:2], first=5)
    st.call(s3, bnn3, num_valid=1)                      # full: dropped, the padding graph not counted
    assert st.cursor.tolist() == [7, 2]
    check_topk(st, s2[:21], bnn2[:2], first=5)


# ---- FusedPredictor -------------------------------------------------------------------------------------------------------
def make_module(engine="tcgen05", style="graph", hidden=32, seed=0, **kw):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, hidden, 4, 2, concat_all_absdf=True, engine=engine, label_style=style, **kw).to(DEV)


def batch_list(seed=0, sizes=(17, 64, 100, 40)):
    return [synth.make_batch(n, 30, seed=seed + i, variable=True, vuln_rate=0.05) for i, n in enumerate(sizes)]


def host_results(pr):
    return {k: v.cpu().numpy() for k, v in pr.results().items()}


def same_results(a, b):
    return sorted(a) == sorted(b) and all(R.same_floats(a[k], b[k]) if a[k].dtype == np.float32 else np.array_equal(a[k], b[k])
                                          for k in a)


def bnn_of(batches):
    return np.concatenate([b.batch_num_nodes().numpy() for b in batches])


@pytest.mark.parametrize("engine,hidden", [("tcgen05", 32), ("simt", 20)])       # W = 128 and W = 80
def test_graph_style_probabilities_are_the_module_sigmoid(engine, hidden):
    m = make_module(engine, "graph", hidden)
    batches = batch_list(1)
    pr = D.FusedPredictor(m, capacity=sum(b.batch_size for b in batches))
    for b in batches:
        pr.predict(b)
    r = pr.results()
    with torch.no_grad():
        x = torch.cat([m(b.to(DEV), {}).reshape(-1) for b in batches])
    # the same forward kernels give the same logits; the store's expression is 1.f / (1.f + expf(-x))
    assert R.same_bits(r["prob"].cpu().numpy(), (1.0 / (1.0 + torch.exp(-x))).cpu().numpy())
    assert set(r) == {"prob"}


@pytest.mark.parametrize("engine,hidden", [("tcgen05", 32), ("simt", 20)])
def test_node_style_probability_is_the_maximum_over_statements(engine, hidden):
    m = make_module(engine, "node", hidden)
    batches = batch_list(2)
    F = sum(b.batch_size for b in batches)
    pr = D.FusedPredictor(m, capacity=F, statements="probability", top_k=10)
    plain = D.FusedPredictor(m, capacity=F)
    ev = D.FusedEvaluator(m, statements="probability")
    scores = []
    for b in batches:
        pr.predict(b)
        plain.predict(b)
        ev.update(b)
        scores.append(ev.last_scores().cpu().numpy().copy())
    s = np.concatenate(scores)
    bnn = bnn_of(batches)
    n0 = np.concatenate([[0], np.cumsum(bnn)])
    want = np.array([s[a:a + n].max() if n else 0.0 for a, n in zip(n0, bnn)], np.float32)
    r = host_results(pr)
    assert R.same_bits(r["prob"], want)
    assert R.same_bits(host_results(plain)["prob"], want)
    want_i, want_s = R.store(s, bnn, 10)
    assert np.array_equal(r["top_statements"], want_i) and R.same_floats(r["top_scores"], want_s)


@pytest.mark.parametrize("engine,hidden", [("tcgen05", 32), ("simt", 20)])
def test_encoder_mode_embeddings_and_attention(engine, hidden):
    m = make_module(engine, "graph", hidden, encoder_mode=True)
    batches = batch_list(3)
    F = sum(b.batch_size for b in batches)
    pr = D.FusedPredictor(m, capacity=F)
    pa = D.FusedPredictor(m, capacity=F, statements="attention", top_k=7)
    for b in batches:
        pr.predict(b)
        pa.predict(b)
    with torch.no_grad():
        want = torch.cat([m(b.to(DEV), {}) for b in batches]).cpu().numpy()
    r, ra = host_results(pr), host_results(pa)
    assert set(r) == {"embedding"} and r["embedding"].shape == (F, m.out_dim)
    assert R.same_bits(r["embedding"], want)
    assert R.same_bits(ra["embedding"], want)
    # the attention of the same encoder under a graph-style head (the head does not enter α)
    g = make_module(engine, "graph", hidden)
    g.load_state_dict(m.state_dict(), strict=False)
    ev = D.FusedEvaluator(g, statements="attention")
    s = []
    for b in batches:
        ev.update(b)
        s.append(ev.last_scores().cpu().numpy().copy())
    want_i, want_s = R.store(np.concatenate(s), bnn_of(batches), 7)
    assert np.array_equal(ra["top_statements"], want_i) and R.same_bits(ra["top_scores"], want_s)


MODES = [("graph", "attention", {}), ("graph", "saliency", {}), ("graph", "integrated_gradients", {"ig_steps": 8}),
         ("graph", "deeplift", {}), ("graph", "deeplift_shap", {"baseline_stdev": 0.5, "shap_samples": 3}),
         ("graph", "gradient_shap", {"noise_stdev": 0.1, "baseline_stdev": 0.2}), ("node", "probability", {})]


@pytest.mark.parametrize("style,mode,kw", MODES, ids=[m[1] for m in MODES])
def test_every_statement_mode_stores_the_evaluator_scores(style, mode, kw):
    m = make_module("tcgen05", style)
    b = synth.make_batch(256, 150, seed=0, variable=True, vuln_rate=0.003 if style == "graph" else 0.06)      # C0
    ev = D.FusedEvaluator(m, statements=mode, **kw)
    pr = D.FusedPredictor(m, capacity=256, statements=mode, top_k=10, **kw)
    for _ in range(3):                                  # eager, capture, replay: the draws advance the same way in both
        ev.update(b)
        s = ev.last_scores().cpu().numpy().copy()
        pr.reset()
        pr.predict(b)
        r = host_results(pr)
        want_i, _ = R.store(s, b.batch_num_nodes().numpy(), 10)
        assert np.array_equal(r["top_statements"], want_i)
        n0 = np.concatenate([[0], np.cumsum(b.batch_num_nodes().numpy())])[:-1]
        ok = want_i >= 0
        assert R.same_bits(r["top_scores"][ok], s[(n0[:, None] + np.maximum(want_i, 0))[ok]])
        assert np.isnan(r["top_scores"][~ok]).all()


@pytest.mark.parametrize("style,mode", [("graph", "attention"), ("node", "probability")])
def test_batch_paths_give_bit_identical_results(style, mode):
    m = make_module("tcgen05", style)
    batches = batch_list(10)              # 100 graphs, not 255: bucketing's padding graph keeps the readout on the same MLP path
    arena = D.GraphArena.from_graphs(batches, device=DEV)
    offs = np.cumsum([0] + [b.batch_size for b in batches])
    dev_batches = [b.to(DEV) for b in batches]
    F = 3 * int(offs[-1])

    def run(fn, passes=3, **kw):
        pr = D.FusedPredictor(m, capacity=F, statements=mode, top_k=10, **kw)
        for _ in range(passes):                          # eager visit, capture, replays
            for i, b in enumerate(batches):
                fn(pr, i, b)
        return pr, host_results(pr)

    _, host = run(lambda pr, i, b: pr.predict(b))
    assert host["prob"].shape == (F,)
    _, eager = run(lambda pr, i, b: pr.predict(b), use_cuda_graph=False)
    res_pr, resident = run(lambda pr, i, b: pr.predict(dev_batches[i]))
    assert len(res_pr._graphs) == len(batches), "one captured graph per resident batch"
    _, ids = run(lambda pr, i, b: pr.predict_ids(arena, np.arange(offs[i], offs[i + 1])))

    def prefetched(pr, i, b):
        if i + 1 < len(batches):
            pr.prefetch(batches[i + 1])
        pr.predict(b)
    _, pre = run(prefetched)
    _, few = run(lambda pr, i, b: pr.predict(b), max_graph_shapes=1)
    _, bucketed = run(lambda pr, i, b: pr.predict(b), bucket_nodes=512, bucket_edges=1024)
    _, bucketed_eager = run(lambda pr, i, b: pr.predict(b), use_cuda_graph=False, bucket_nodes=512)
    for name, r in (("eager", eager), ("resident", resident), ("ids", ids), ("prefetch", pre), ("max_graph_shapes=1", few),
                    ("bucketed", bucketed), ("bucketed eager", bucketed_eager)):
        assert same_results(r, host), name


def test_batches_without_labels():
    m = make_module("tcgen05", "graph")
    sizes = (30, 50)
    labelled = batch_list(20, sizes)
    bare = batch_list(20, sizes)
    for b in bare:
        b.ndata.pop("_VULN")
    F = sum(sizes)
    out = []
    for batches in (labelled, bare):
        host = D.FusedPredictor(m, capacity=2 * F, statements="saliency", top_k=5)
        arena = D.GraphArena.from_graphs(batches, device=DEV)
        ids = D.FusedPredictor(m, capacity=2 * F, statements="saliency", top_k=5)
        for _ in range(2):
            for b in batches:
                host.predict(b)
            ids.predict_ids(arena, np.arange(F))
        out.append((host_results(host), host_results(ids)))
    assert same_results(out[0][0], out[1][0]) and same_results(out[0][1], out[1][1])


def test_parameters_and_grads_stay_and_training_is_followed():
    m = make_module("tcgen05", "graph", seed=3)
    for p in m.parameters():
        p.grad = torch.randn_like(p)
    before = [(p.detach().clone(), p.grad.clone()) for p in m.parameters()]
    batches = batch_list(30)
    pr = D.FusedPredictor(m, capacity=1000, statements="deeplift")
    for _ in range(2):
        for b in batches:
            pr.predict(b)
    pr.results()
    for p, (v, g) in zip(m.parameters(), before):
        assert torch.equal(p.detach(), v) and torch.equal(p.grad, g)
    for p in m.parameters():
        p.grad = None
    tr = D.FusedTrainer(m, use_cuda_graph=True, distributed=False)
    for i in range(2):
        tr.step(synth.make_batch(32, 30, seed=100 + i, variable=True, vuln_rate=0.01))
    pr.reset()
    for b in batches:
        pr.predict(b)
    with torch.no_grad():
        x = torch.cat([m(b.to(DEV), {}).reshape(-1) for b in batches])
    assert R.same_bits(pr.results()["prob"].cpu().numpy(), (1.0 / (1.0 + torch.exp(-x))).cpu().numpy())


def test_reset_overflow_and_bad_indices():
    m = make_module("simt", "graph")
    b = synth.make_batch(16, 20, seed=1)
    pr = D.FusedPredictor(m, capacity=20, statements="attention", top_k=3)
    pr.predict(b)
    first = host_results(pr)
    pr.predict(b)
    with pytest.raises(ValueError, match="capacity >= 32"):
        pr.results()
    pr.reset()
    pr.predict(b)
    assert same_results(host_results(pr), first)
    bad = synth.make_batch(8, 20, seed=2)
    bad.ndata[next(k for k in bad.ndata if k != "_VULN")][3] = 5000
    pr.predict(bad)
    with pytest.raises(IndexError):
        pr.results()


@pytest.mark.parametrize("det", ["1", None])
def test_runs_are_bit_identical(det, monkeypatch):
    if det is None:
        monkeypatch.delenv("DDFA_DETERMINISTIC", raising=False)
    else:
        monkeypatch.setenv("DDFA_DETERMINISTIC", det)
    _lib.apply_deterministic_mode()
    runs = []
    for _ in range(2):
        m = make_module("tcgen05", "graph", seed=9)
        pr = D.FusedPredictor(m, capacity=1000, statements="attention", top_k=10)
        for _ in range(2):
            for b in batch_list(40):
                pr.predict(b)
        runs.append(host_results(pr))
    assert same_results(runs[0], runs[1])
