"""GPU: DeepLift, DeepLiftShap and GradientShap statement scores of FusedEvaluator.  The per-node scores against the fp64 oracle
(tests/attribution_rule.py) on both engines, at several widths and head depths, on C0- and C1-size batches; ddfa_stmt_shap_input's
draws against the host Philox; deeplift_shap at baseline_stdev = 0 bit-identical to deeplift; host, eager, resident, arena,
prefetched and bucketed runs bit-identical; deterministic repeats; the batch counter and the statement metric keys."""
import os
import sys

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from oracle import ggnn_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attribution_rule as A  # noqa: E402
import statement_rule as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
# relative to the largest |score|: the bounds test_statements_gpu.py holds saliency and integrated gradients to
GRAD_TOL = {"simt": 2e-4, "tcgen05": 2e-3}
SEED = 12345


def make_pair(engine, hidden, layers, seed=0):
    torch.manual_seed(seed)
    o = O.OracleFlowGNNGGNN(FEAT, 1002, hidden, 4, layers, concat_all_absdf=True)
    m = D.FlowGNNGGNNModule(FEAT, 1002, hidden, 4, layers, concat_all_absdf=True, engine=engine)
    m.load_state_dict(o.state_dict())
    return m.to(DEV), o.double()


def c0(seed=0):
    return synth.make_batch(256, 150, seed=seed, variable=True, vuln_rate=0.3)


def c1(seed=0):
    return synth.make_batch(1024, 150, seed=seed, variable=True, vuln_rate=0.3)


def scores_of(ev, b):
    ev.update(b)
    torch.cuda.synchronize()
    return ev.last_scores().clone()


def oracle_scores(o, b, mode, samples, baseline_stdev, noise_stdev, batch=0):
    if mode == "gradient_shap":
        return A.oracle_gradient_shap(o, b, SEED, batch, samples, noise_stdev, baseline_stdev)
    with torch.no_grad():
        x = o.embed(b)
    if mode == "deeplift" or baseline_stdev == 0:
        return A.oracle_deeplift(o, b, [torch.zeros_like(x)])
    N, Dm = x.shape
    return A.oracle_deeplift(o, b, [baseline_stdev * torch.from_numpy(A.gaussians(SEED, batch, j, N, Dm, True))
                                    for j in range(samples)])


# (engine, W, head layers, batch): W = 4 * hidden (four embedding tables)
ORACLE_CASES = [("simt", 32, 1, "c0"), ("simt", 32, 2, "c0"), ("simt", 32, 3, "c0"),
                ("tcgen05", 128, 1, "c0"), ("tcgen05", 128, 2, "c0"), ("tcgen05", 128, 3, "c0"),
                ("tcgen05", 256, 2, "c0"), ("tcgen05", 128, 2, "c1")]
MODES = [("deeplift", {}), ("deeplift_shap", dict(shap_samples=2, baseline_stdev=0.5)),
         ("gradient_shap", dict(shap_samples=2, baseline_stdev=0.25, noise_stdev=0.1))]


@pytest.mark.parametrize("engine,W,layers,size", ORACLE_CASES)
def test_scores_match_the_oracle(engine, W, layers, size):
    m, o = make_pair(engine, W // 4, layers, seed=W + layers)
    b = c0(seed=1) if size == "c0" else c1(seed=2)
    modes = MODES if size == "c0" else MODES[:1]
    vuln = b.ndata["_VULN"].numpy()
    for mode, kw in modes:
        ev = D.FusedEvaluator(m, statements=mode, attribution_seed=SEED, **kw)
        got = scores_of(ev, b).cpu().double()
        assert got.numel() == b.num_nodes() and ev.attribution_draws == 1
        ref = oracle_scores(o, b, mode, kw.get("shap_samples", 1), kw.get("baseline_stdev", 0.0), kw.get("noise_stdev", 0.0))
        err = float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
        print(f"{engine}/W={W}/L={layers}/{size} {mode}: max deviation {err:.2e} of max |score| {float(ref.abs().max()):.3e}")
        assert err <= GRAD_TOL[engine], (mode, err)
        st = ev.statement_state().cpu().numpy()
        assert np.array_equal(st, R.host_state(got.float().numpy(), vuln, b.batch_num_nodes().numpy(), False)), mode
        r = ev.compute("test_")
        assert r["test_stmt_functions"] == b.batch_size and "test_stmt_top1" in r and "test_stmt_ifa" in r
        assert "test_stmt_all_top1" not in r


def test_deeplift_shap_at_zero_stdev_is_deeplift_bit_for_bit():
    m, _ = make_pair("tcgen05", 32, 3, seed=3)
    b = c0(seed=4)
    a = scores_of(D.FusedEvaluator(m, statements="deeplift"), b)
    s = scores_of(D.FusedEvaluator(m, statements="deeplift_shap"), b)
    s16 = scores_of(D.FusedEvaluator(m, statements="deeplift_shap", shap_samples=16, attribution_seed=9), b)
    assert torch.equal(a, s) and torch.equal(a, s16)


def _shap_input(x, gp, alpha, noise, base, seed, counter, sample, image=None):
    N, Dm = x.shape
    inp, diff = torch.empty_like(x), torch.empty_like(x)
    _lib.lib().call("ddfa_stmt_shap_input", x.data_ptr(), gp.data_ptr(), gp.numel() - 1, N, Dm, float(alpha), float(noise), float(base),
                    seed, counter.data_ptr(), sample, inp.data_ptr(), diff.data_ptr(), 0 if image is None else image.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return inp, diff


def test_shap_input_draws_match_the_host():
    b = c0(seed=5)
    bnn = b.batch_num_nodes()
    gp = torch.as_tensor(np.concatenate([[0], np.cumsum(bnn.numpy())]).astype(np.int32)).to(DEV)
    N, Dm = b.num_nodes(), 128
    x = torch.randn(N, Dm, device=DEV)
    counter = torch.tensor([7], dtype=torch.int64, device=DEV)
    gid = torch.repeat_interleave(torch.arange(bnn.numel()), bnn).to(DEV)
    seed = 2 ** 63 + 11
    # alpha drawn per function, zero baseline, no noise: input = fp32(alpha_b * x) exactly, diff = x
    inp, diff = _shap_input(x, gp, -1.0, 0.0, 0.0, seed, counter, 3)
    alpha = torch.from_numpy(A.alphas(seed, 7, 3, bnn.numel())).to(DEV)[gid][:, None]
    assert torch.equal(diff, x) and torch.equal(inp, alpha * x)
    # alpha = 0 writes the baseline itself; the Gaussians agree with the host's fp64 Box-Muller to fp32 rounding
    inp, diff = _shap_input(x, gp, 0.0, 0.5, 2.0, seed, counter, 1)
    noise = torch.from_numpy(A.gaussians(seed, 7, 1, N, Dm, False)).to(DEV)
    base = torch.from_numpy(A.gaussians(seed, 7, 1, N, Dm, True)).to(DEV)
    assert float((inp.double() - 2.0 * base).abs().max()) <= 1e-5
    assert float((diff.double() - (x.double() + 0.5 * noise - 2.0 * base)).abs().max()) <= 1e-5
    # the activation image is that of the written rows
    nbytes = _lib.lib().call("ddfa_act_image_bytes", N)
    img, want = torch.zeros(nbytes, dtype=torch.uint8, device=DEV), torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    inp, _ = _shap_input(x, gp, -1.0, 0.1, 0.3, seed, counter, 0, image=img)
    _lib.lib().call("ddfa_act_to_image", inp.data_ptr(), N, Dm, want.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(img, want)
    assert int(counter.item()) == 7       # read, not advanced


PATH_MODES = [("deeplift", {}), ("deeplift_shap", dict(shap_samples=3, baseline_stdev=0.5)),
              ("gradient_shap", dict(shap_samples=3, baseline_stdev=0.2, noise_stdev=0.1))]


@pytest.mark.parametrize("mode,kw", PATH_MODES, ids=[p[0] for p in PATH_MODES])
def test_paths_give_bit_identical_scores_and_state(mode, kw):
    m, _ = make_pair("tcgen05", 32, 3, seed=6)
    # below 256 graphs with the padding graph too: the head runs the same in-CTA form bucketed or not (at 256 and more it runs the
    # batched GEMM form, whose hidden activations differ in the last bits, and the rescale multipliers follow them)
    batches = [synth.make_batch(n, 60, seed=10 + i, variable=True, vuln_rate=0.3) for i, n in enumerate((17, 64, 200))]
    arena = D.GraphArena.from_graphs(batches, device=DEV)
    offs = np.cumsum([0] + [b.batch_size for b in batches])
    dev_batches = [b.to(DEV) for b in batches]

    def run(fn, ev, passes=2):
        out = []
        for _ in range(passes):
            for i, b in enumerate(batches):
                fn(ev, i, b)
                torch.cuda.synchronize()
                out.append(ev.last_scores().clone())
        assert ev.attribution_draws == passes * len(batches)
        return out, ev.statement_state().clone()

    kw = dict(statements=mode, attribution_seed=SEED, **kw)
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
    if mode != "deeplift":       # fresh draws on every replay: the second pass differs from the first
        assert not torch.equal(host[0][0], host[0][3])
    else:
        assert torch.equal(host[0][0], host[0][3])
    bkw = dict(bucket_nodes=512, bucket_edges=1024, **kw)
    bucketed = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, **bkw))
    bucketed_eager = run(lambda ev, i, b: ev.update(b), D.FusedEvaluator(m, use_cuda_graph=False, **bkw))
    assert torch.equal(bucketed[1], bucketed_eager[1])
    for a, b, h in zip(bucketed[0], bucketed_eager[0], host[0]):
        assert torch.equal(a, b) and a.shape == h.shape
    # the counter can be set back: the same batch at the same count draws the same values
    ev = D.FusedEvaluator(m, **kw)
    first = scores_of(ev, batches[1])
    scores_of(ev, batches[1])
    ev.attribution_draws = 0
    assert torch.equal(scores_of(ev, batches[1]), first)


@pytest.mark.parametrize("mode,kw", PATH_MODES[1:], ids=[p[0] for p in PATH_MODES[1:]])
def test_deterministic_repeats_and_nothing_is_written(mode, kw, monkeypatch):
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
    m, _ = make_pair("tcgen05", 32, 2, seed=8)
    b = c1(seed=9)
    for p in m.parameters():
        p.grad = torch.full_like(p, 0.25)
    before = [p.detach().clone() for p in m.parameters()]
    runs = []
    for _ in range(2):
        ev = D.FusedEvaluator(m, statements=mode, attribution_seed=SEED, **kw)
        runs.append((scores_of(ev, b), ev.statement_state().clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    for p, q in zip(m.parameters(), before):
        assert torch.equal(p.detach(), q) and bool((p.grad == 0.25).all())
