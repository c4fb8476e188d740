"""GPU: the threshold curves (ddfa_curve_sort / ddfa_curve_metrics, binary_curves, FusedEvaluator.curves) against the NumPy
restatement of torchmetrics < 0.10 (tests/curve_rule.py) and scikit-learn: thresholds bit for bit, counts exact, fp64 ratios
equal, AUROC and average precision within 1e-12; sizes past 2^24 samples, heavy ties, signed zeros and subnormals; the
evaluator's host and arena paths; the error rules; bit-reproducibility in both deterministic modes."""
import os
import sys

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200.evaluator import binary_curves

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import curve_rule as R  # noqa: E402
import nonfinite_sites as NS  # noqa: E402

sklearn_metrics = pytest.importorskip("sklearn.metrics")

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
KEYS = ("pr_curve", "roc_curve", "pr_curve_binned", "AUROC", "AveragePrecision")


def bits(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def inputs(kind: str, n: int, seed: int = 0):
    """(probs, labels) as fp32 NumPy arrays: about 6 % positives, both classes present from n = 2 on (but "one_positive")."""
    rng = np.random.default_rng(seed)
    y = (rng.random(n) < 0.06).astype(np.float32)
    if kind == "uniform":
        p = rng.random(n, dtype=np.float32)
    elif kind == "quantised":
        p = (np.floor(rng.random(n) * 256) / 256).astype(np.float32)        # multiples of 2^-8: massive ties
    elif kind == "equal":
        p = np.full(n, 0.375, np.float32)
    elif kind == "zero_one":
        p = rng.choice(np.float32([0, 1]), n)
    elif kind == "signed_zero":
        p = rng.choice(np.float32([-0.0, 0.0, 0.5, 1e-30]), n)
    elif kind == "subnormal":
        p = rng.choice(np.array([0, 1, 2, 3, 0x400000, 0x7FFFFF, 0x800000, 0x80000001], np.uint32).view(np.float32), n)
    elif kind == "one_positive":
        p = rng.random(n, dtype=np.float32)
        y[:] = 0
        y[rng.integers(n)] = 1
    else:
        raise ValueError(kind)
    if n >= 2 and kind != "one_positive":
        y[:2] = [1, 0]
    return p, y


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def raw(p, y, bins):
    """Both entry points through the ABI, every output cut to the lengths of the info words (unwritten entries hold -7)."""
    n = p.numel()
    L = _lib.lib()
    ws = torch.empty(L.call("ddfa_curve_workspace_bytes", n), dtype=torch.uint8, device=DEV)

    def e(k, dt):
        return torch.full((k,), -7, dtype=dt, device=DEV)
    thr, tps, fps, info = e(n, torch.float32), e(n, torch.int64), e(n, torch.int64), e(_lib.CURVE_INFO_WORDS, torch.int64)
    pr_p, pr_r, fpr, tpr = (e(n + 1, torch.float64) for _ in range(4))
    pr_t, roc_t = e(n, torch.float32), e(n + 1, torch.float32)
    b = dev(np.float32(bins))
    bp, br, summary = e(b.numel() + 1, torch.float64), e(b.numel() + 1, torch.float64), e(2, torch.float64)
    st = torch.cuda.current_stream().cuda_stream
    L.call("ddfa_curve_sort", p.data_ptr(), y.data_ptr(), n, thr.data_ptr(), tps.data_ptr(), fps.data_ptr(), info.data_ptr(),
           ws.data_ptr(), ws.numel(), st)
    L.call("ddfa_curve_metrics", thr.data_ptr(), tps.data_ptr(), fps.data_ptr(), n, b.data_ptr(), b.numel(), pr_p.data_ptr(),
           pr_r.data_ptr(), pr_t.data_ptr(), fpr.data_ptr(), tpr.data_ptr(), roc_t.data_ptr(), bp.data_ptr(), br.data_ptr(),
           summary.data_ptr(), info.data_ptr(), ws.data_ptr(), ws.numel(), st)
    torch.cuda.synchronize()
    w = info.cpu().tolist()
    m, k = w[0], w[1]
    c = lambda t: t.cpu().numpy()     # noqa: E731
    return dict(info=w, thr=c(thr[:m]), tps=c(tps[:m]), fps=c(fps[:m]), pr=(c(pr_p[:k + 1]), c(pr_r[:k + 1]), c(pr_t[:k])),
                roc=(c(fpr[:m + 1]), c(tpr[:m + 1]), c(roc_t[:m + 1])), binned=(c(bp), c(br)), summary=summary.cpu().tolist(),
                untouched=(c(thr[m:]), c(tps[m:])))


def check_raw(r, p, y, bins):
    thr, tps, fps = R.clf_curve(p, y)
    P = int(np.count_nonzero(y == 1))
    assert r["info"][:7] == [len(thr), len(R.pr_curve(p, y)[2]), P, len(p) - P, 0, 0, int(P == 0 or P == len(p))]
    assert np.array_equal(bits(r["thr"]), bits(thr))
    assert np.array_equal(r["tps"], tps) and np.array_equal(r["fps"], fps)
    assert np.all(bits(r["untouched"][0]) == bits(-7.0)) and np.all(r["untouched"][1] == -7)
    want = R.pr_curve(p, y)
    np.testing.assert_array_equal(r["pr"][0], want[0])
    np.testing.assert_array_equal(r["pr"][1], want[1])
    assert np.array_equal(bits(r["pr"][2]), bits(want[2]))
    want = R.roc_curve(p, y)
    np.testing.assert_array_equal(r["roc"][0], want[0])
    np.testing.assert_array_equal(r["roc"][1], want[1])
    assert np.array_equal(bits(r["roc"][2]), bits(want[2]))
    want = R.binned(p, y, bins)
    np.testing.assert_array_equal(r["binned"][0], want[0])
    np.testing.assert_array_equal(r["binned"][1], want[1])


def check_public(out, p, y, bins=None):
    """binary_curves' result against the restatement (exact) and scikit-learn (AUROC / AP within 1e-12 relative)."""
    bins = R.default_bins() if bins is None else np.float32(bins)
    assert set(out) == set(KEYS)
    got = [tuple(t.cpu().numpy() for t in out[k]) for k in KEYS[:3]]
    for (gp, gr, gt), (wp, wr, wt) in zip(got, (R.pr_curve(p, y), R.roc_curve(p, y), R.binned(p, y, bins))):
        assert gp.dtype == np.float64 and gr.dtype == np.float64 and gt.dtype == np.float32
        np.testing.assert_array_equal(gp, wp)
        np.testing.assert_array_equal(gr, wr)
        assert np.array_equal(bits(gt), bits(wt))
    assert out["AUROC"] == pytest.approx(sklearn_metrics.roc_auc_score(y, p), rel=1e-12, abs=0)
    assert out["AveragePrecision"] == pytest.approx(sklearn_metrics.average_precision_score(y, p), rel=1e-12, abs=0)
    pr = R.pr_curve(p, y)
    assert out["AveragePrecision"] == pytest.approx(R.average_precision(pr[0], pr[1]), rel=1e-12, abs=0)
    roc = R.roc_curve(p, y)
    assert out["AUROC"] == pytest.approx(R.auroc(roc[0], roc[1]), rel=1e-12, abs=0)


# ---- the kernels and binary_curves against the restatement ------------------------------------------------------------------
def test_hand_computed_case():
    p, y = np.float32([.9, .8, .8, .3, .2, .7, .1, .1]), np.float32([1, 0, 1, 0, 0, 1, 0, 0])
    out = binary_curves(dev(p), dev(y))
    prec, rec, thr = (t.cpu().numpy() for t in out["pr_curve"])
    assert thr.tolist() == np.float32([.7, .8, .9]).tolist()
    assert prec.tolist() == [.75, 2 / 3, 1, 1] and rec.tolist() == [1, 2 / 3, 1 / 3, 0]
    assert out["AveragePrecision"] == pytest.approx(0.80556, abs=5e-6) and out["AUROC"] == pytest.approx(0.9, abs=1e-15)
    check_public(out, p, y)


@pytest.mark.parametrize("n", [1, 2, 19_000, 1_000_000, 2 ** 24 + 3])
def test_sizes(n):
    """2^24 + 3 samples: a count held in fp32 anywhere would round."""
    p, y = inputs("uniform", n, seed=n)
    bins = R.default_bins()
    check_raw(raw(dev(p), dev(y), bins), p, y, bins)
    if n == 1:
        with pytest.raises(ValueError, match="only one class"):
            binary_curves(dev(p), dev(y))
        return
    check_public(binary_curves(dev(p), dev(y)), p, y)


@pytest.mark.parametrize("kind", ["quantised", "equal", "zero_one", "signed_zero", "subnormal", "one_positive"])
@pytest.mark.parametrize("n", [19_000, 1_000_000])
def test_inputs(kind, n):
    p, y = inputs(kind, n, seed=7)
    bins = R.default_bins()
    r = raw(dev(p), dev(y), bins)
    check_raw(r, p, y, bins)
    if kind == "signed_zero":
        assert 0.0 in r["thr"].tolist() and not np.any(bits(r["thr"]) == 0x80000000)     # -0.0 tied with +0.0, shown as +0.0
    check_public(binary_curves(dev(p), dev(y)), p, y)


def test_custom_bins_and_a_side_stream():
    p, y = inputs("quantised", 50_000, seed=3)
    bins = [0.0, 0.25, 0.5, 0.5, 0.75, 1.0, 2.0]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = binary_curves(dev(p), dev(y), binned_thresholds=bins)
    check_public(out, p, y, bins)
    assert out["pr_curve_binned"][2].cpu().tolist() == bins


# ---- through the evaluator -------------------------------------------------------------------------------------------------
def make_module(engine, style, seed=0):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine, label_style=style).to(DEV)


def c0_batches(style):
    """Three C0-size batches (256 graphs of about 150 nodes) with one vulnerable statement in each vulnerable function: about
    6 % vulnerable functions in graph style, half of them in node style (about 0.3 % positive statements)."""
    rate = 0.06 if style == "graph" else 0.5
    return [synth.make_batch(256, 150, seed=40 + i, variable=True, vuln_rate=rate) for i in range(3)]


@pytest.mark.parametrize("style", ["graph", "node"])
def test_evaluator_curves_on_host_batches_and_an_arena(style):
    m = make_module("tcgen05", style)
    batches = c0_batches(style)
    total = sum(b.batch_size if style == "graph" else b.num_nodes() for b in batches)
    arena = D.GraphArena.from_graphs(batches, device=DEV)
    offs = np.cumsum([0] + [b.batch_size for b in batches])
    runs = {"host": lambda ev: [ev.update(b) for b in batches],
            "arena": lambda ev: [ev.update_ids(arena, np.arange(offs[i], offs[i + 1])) for i in range(len(batches))]}
    for path, run in runs.items():
        ev = D.FusedEvaluator(m, max_predictions=total)
        run(ev)
        before = ev.compute("test_")
        cur = ev.curves("test_")
        assert ev.compute("test_") == before, path
        assert set(cur) == {f"test_{k}" for k in KEYS}
        probs, labels = ev.predictions()
        assert probs.numel() == total
        direct = binary_curves(probs, labels)
        for k in KEYS[:3]:
            for a, b in zip(cur[f"test_{k}"], direct[k]):
                assert torch.equal(a, b), (path, k)
        assert cur["test_AUROC"] == direct["AUROC"] and cur["test_AveragePrecision"] == direct["AveragePrecision"]
        p, y = probs.cpu().numpy(), labels.cpu().numpy()
        print(f"{style}/{path}: {total} samples, {int(y.sum())} positive, {len(cur['test_roc_curve'][2]) - 1} distinct thresholds, "
              f"AUROC {cur['test_AUROC']:.6f}, AP {cur['test_AveragePrecision']:.6f}")
        check_public(direct, p, y)
        assert ev.curves("val_", binned_thresholds=10)["val_pr_curve_binned"][2].numel() == 10


def test_evaluator_curves_raise_as_compute_does():
    m = make_module("simt", "graph")
    b = synth.make_batch(16, 20, seed=1, vuln_rate=0.3)
    with pytest.raises(ValueError, match="max_predictions=0"):
        ev = D.FusedEvaluator(m)
        ev.update(b)
        ev.curves()
    ev = D.FusedEvaluator(m, max_predictions=10)
    with pytest.raises(ValueError, match="no sample"):
        ev.curves()
    ev.update(b)
    with pytest.raises(ValueError, match="max_predictions >= 16"):
        ev.curves()
    clean = D.FusedEvaluator(m, max_predictions=16)
    clean.update(synth.make_batch(16, 20, seed=1, vuln_rate=0.0))
    with pytest.raises(ValueError, match=r"only one class present \(0 positives, 16 negatives\)"):
        clean.curves()


def test_nan_logit_raises_with_the_count():
    g, where = NS.poison_batch("graph", 64, seed=2)
    m = make_module("simt", "graph")
    with torch.no_grad():
        dict(m.named_parameters())[NS.EMBED][where["row"]] = float("nan")
    ev = D.FusedEvaluator(m, max_predictions=64)
    ev.update(g)
    probs, _ = ev.predictions()
    assert int(torch.isnan(probs).sum()) == 1
    with pytest.raises(ValueError, match="1 of 64 probabilities are NaN"):
        ev.curves()


def test_binary_curves_error_paths():
    p, y = dev(np.float32([.1, .9, .5])), dev(np.float32([0, 1, 1]))
    with pytest.raises(ValueError, match="no samples"):
        binary_curves(p[:0], y[:0])
    with pytest.raises(ValueError, match="2 of 3 labels are neither 0 nor 1"):
        binary_curves(p, dev(np.float32([0, 2, np.nan])))
    with pytest.raises(ValueError, match="only one class"):
        binary_curves(p, dev(np.float32([1, 1, 1])))
    with pytest.raises(ValueError, match="1 of 3 probabilities are NaN"):
        binary_curves(dev(np.float32([.1, np.nan, .5])), y)
    with pytest.raises(ValueError, match="1-D float32"):
        binary_curves(p.double(), y)
    with pytest.raises(ValueError, match="differ"):
        binary_curves(p, y[:2])
    with pytest.raises(_lib.DdfaError, match="CUDA tensor"):
        binary_curves(p.cpu(), y)
    with pytest.raises(ValueError, match="binned_thresholds"):
        binary_curves(p, y, binned_thresholds=0)


def test_bit_reproducible_in_both_deterministic_modes():
    L = _lib.lib()
    old = L.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC)
    p, y = inputs("quantised", 1_000_003, seed=5)
    results = []
    try:
        for det in (0, 1, 0, 1):
            L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, det)
            results.append(binary_curves(dev(p), dev(y)))
    finally:
        L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, old)
    a = results[0]
    for b in results[1:]:
        for k in KEYS[:3]:
            for s, t in zip(a[k], b[k]):
                assert torch.equal(s, t), k
        assert np.float64(a["AUROC"]).tobytes() == np.float64(b["AUROC"]).tobytes()
        assert np.float64(a["AveragePrecision"]).tobytes() == np.float64(b["AveragePrecision"]).tobytes()
