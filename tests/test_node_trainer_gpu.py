"""GPU: label_style="node" in FusedTrainer — the device sampler of the loss rows (ddfa_node_sample), the head over a row list
(ddfa_node_head_fwd / ddfa_node_bce / ddfa_node_head_bwd) against fp64, and the trainer against the module path fed the same
rows (module.forward + module.loss_fn + backward + torch.optim.Adam)."""
import copy
import itertools

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200 import engine as E

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


# ---- the sampler, through the ABI ----------------------------------------------------------------------------------------
class Sampler:
    def __init__(self, vuln, n_valid, seed=5):
        self.vuln = torch.as_tensor(vuln, dtype=torch.int32).to(DEV)
        N = self.vuln.numel()
        self.valid = torch.tensor([n_valid], dtype=torch.int32, device=DEV)
        self.rows = torch.full((N,), -1, dtype=torch.int32, device=DEV)
        self.S = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.status = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.draw = torch.zeros(1, dtype=torch.int64, device=DEV)
        self.seed = seed

    def __call__(self, factor):
        with torch.cuda.device(DEV):
            E.node_sample(self.vuln, self.valid, factor, self.seed, self.draw, self.rows, self.S, self.status)
        return self.rows[: int(self.S.item())].cpu().long()


def random_vuln(N, rate, seed):
    rng = np.random.default_rng(seed)
    return (rng.random(N) < rate).astype(np.int32)


@pytest.mark.parametrize("N,n_valid,factor", [(5000, 4500, 1.5), (5000, 5000, 0.0), (1024, 1000, 2.0), (157381, 150000, 1.0), (3, 3, 0.5)])
def test_sampler_rows(N, n_valid, factor):
    vuln = random_vuln(N, 0.1, N)
    vuln[-1] = 1                                      # a vulnerable padding node (when there is padding) must not appear
    s = Sampler(vuln, n_valid)
    rows = s(factor)
    valid = vuln[:n_valid]
    n_vuln, pop = int(valid.sum()), int((valid == 0).sum())
    k = E.undersample_count(n_vuln, factor)
    assert k <= pop
    assert rows.numel() == n_vuln + k
    assert bool((rows[1:] > rows[:-1]).all()), "ascending and unique"
    assert rows.numel() == 0 or int(rows.max()) < n_valid
    assert set(np.nonzero(valid)[0].tolist()) <= set(rows.tolist())
    assert int(s.status.item()) == 0 and int(s.draw.item()) == 1


def test_sampler_clamps_and_flags_an_oversized_draw():
    vuln = random_vuln(2000, 0.3, 1)
    s = Sampler(vuln, 1900)
    rows = s(100.0)
    assert rows.tolist() == list(range(1900)) and int(s.status.item()) == 1
    rows = s(0.5)
    assert int(s.status.item()) == 1, "the call never clears the status word"


def test_sampler_without_undersampling_takes_every_valid_node():
    s = Sampler(random_vuln(3000, 0.2, 2), 2777)
    assert s(None).tolist() == list(range(2777))
    assert int(s.draw.item()) == 0 and int(s.status.item()) == 0


def test_sampler_same_draw_same_rows_and_consecutive_draws_differ():
    vuln = random_vuln(20000, 0.05, 3)
    s = Sampler(vuln, 20000)
    a, b = s(1.0), s(1.0)
    assert not torch.equal(a, b)
    s.draw.fill_(0)
    assert torch.equal(s(1.0), a)
    assert not torch.equal(Sampler(vuln, 20000, seed=6)(1.0), a)


def test_sampler_subsets_are_uniform():
    """Population 6, k = 2: the 15 subsets over 6 000 consecutive draws (seeded: the test is deterministic)."""
    from scipy.stats import chisquare
    vuln = np.array([0, 1, 0, 0, 1, 0, 0, 0], dtype=np.int32)
    s = Sampler(vuln, 8, seed=11)
    draws = 6000
    out = torch.empty(draws, 4, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        for i in range(draws):
            E.node_sample(s.vuln, s.valid, 1.0, s.seed, s.draw, s.rows, s.S, s.status)
            out[i].copy_(s.rows[:4])
    assert int(s.S.item()) == 4
    out = out.cpu().numpy()
    pop = [0, 2, 3, 5, 6, 7]
    subsets = {c: i for i, c in enumerate(itertools.combinations(pop, 2))}
    counts = np.zeros(len(subsets))
    for r in out:
        assert 1 in r and 4 in r
        counts[subsets[tuple(int(v) for v in r if v not in (1, 4))]] += 1
    stat, p = chisquare(counts)
    print("subset counts", counts.tolist(), "p =", p)
    assert p > 1e-3


def test_sampler_inclusion_frequencies_at_c1_size():
    N = 153600
    vuln = random_vuln(N, 0.1, 4)
    n_vuln, pop = int(vuln.sum()), int((vuln == 0).sum())
    factor = 0.5 * pop / n_vuln
    k = E.undersample_count(n_vuln, factor)
    s = Sampler(vuln, N, seed=9)
    draws = 200
    hits = torch.zeros(N, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        for _ in range(draws):
            E.node_sample(s.vuln, s.valid, factor, s.seed, s.draw, s.rows, s.S, s.status)
            hits[s.rows[: n_vuln + k].long()] += 1
    assert int(s.S.item()) == n_vuln + k
    hits = hits.cpu().numpy()
    assert (hits[vuln == 1] == draws).all()
    p = k / pop
    freq = hits[vuln == 0] / draws
    sigma = (p * (1 - p) / draws) ** 0.5
    print(f"k/M = {p:.4f}, frequencies in [{freq.min():.3f}, {freq.max():.3f}], 5 sigma = {5 * sigma:.3f}")
    assert np.abs(freq - p).max() <= 5 * sigma


# ---- the head, against fp64 ------------------------------------------------------------------------------------------------
def head_case(N, D, L, rows, seed=0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(N, D, generator=g)
    x = torch.randn(N, D, generator=g)
    ws = [torch.randn(2 * D if i < L - 1 else 1, 2 * D, generator=g) / (2 * D) ** 0.5 for i in range(L)]
    bs = [torch.randn(2 * D if i < L - 1 else 1, generator=g) * 0.1 for i in range(L)]
    return h, x, ws, bs, torch.as_tensor(rows, dtype=torch.int32)


def run_head(h, x, ws, bs, rows, dlogits_host):
    N, D = h.shape
    L = len(ws)
    dev = lambda t: t.to(DEV).contiguous()
    params = E.ParamPack([], None, None, None, None, None, None, None, None, [dev(w) for w in ws], [dev(b) for b in bs])
    grads = E.ParamPack([], None, None, None, None, None, None, None, None, [torch.zeros_like(w) for w in params.mlp_w],
                        [torch.zeros_like(b) for b in params.mlp_b])
    rows_d = torch.zeros(N, dtype=torch.int32, device=DEV)
    rows_d[: rows.numel()] = rows.to(DEV)
    S = torch.tensor([rows.numel()], dtype=torch.int32, device=DEV)
    hd, xd = dev(h), dev(x)
    with torch.cuda.device(DEV):
        logits, act = E.node_head_fwd(params, xd, hd, rows_d, S)
        dl = torch.zeros(N, device=DEV)
        dl[: rows.numel()] = dlogits_host.to(DEV)
        dh, dx = E.node_head_bwd(params, grads, dl, xd, hd, rows_d, S, act)
    torch.cuda.synchronize()
    return logits[: rows.numel()].cpu(), dh.cpu(), dx.cpu(), [t.cpu() for t in grads.mlp_w], [t.cpu() for t in grads.mlp_b]


def ref_head(h, x, ws, bs, rows, dlogits):
    o = torch.cat([h, x], 1).double()[rows.long()].requires_grad_(True)
    w64 = [w.double().requires_grad_(True) for w in ws]
    b64 = [b.double().requires_grad_(True) for b in bs]
    a = o
    for i in range(len(ws)):
        a = a @ w64[i].t() + b64[i]
        if i < len(ws) - 1:
            a = torch.relu(a)
    logits = a.reshape(-1)
    logits.backward(dlogits.double())
    D = h.shape[1]
    dh = torch.zeros(h.shape, dtype=torch.float64)
    dx = torch.zeros(h.shape, dtype=torch.float64)
    dh[rows.long()] = o.grad[:, :D]
    dx[rows.long()] = o.grad[:, D:]
    return logits.detach(), dh, dx, [w.grad for w in w64], [b.grad for b in b64]


def close(got, ref, tol=2e-4):
    err = float((got.double() - ref).abs().max()) if ref.numel() else 0.0
    absmax = float(ref.abs().max()) if ref.numel() else 0.0
    assert err < tol * absmax + 1e-6, (err, absmax)


@pytest.mark.parametrize("N,D,L,which", [(1000, 32, 3, "random"), (1000, 32, 3, "empty"), (1000, 128, 2, "one"), (777, 20, 2, "all"),
                                         (157381, 32, 3, "random"), (157381, 16, 1, "all"), (300, 128, 4, "random")])
def test_head_matches_fp64(N, D, L, which):
    rng = np.random.default_rng(N + D + L)
    rows = {"random": np.sort(rng.choice(N, size=N // 7, replace=False)), "empty": np.zeros(0, dtype=np.int64),
            "one": np.array([N // 2]), "all": np.arange(N)}[which]
    h, x, ws, bs, rows = head_case(N, D, L, rows)
    dl = torch.randn(rows.numel(), generator=torch.Generator().manual_seed(1)) / max(1, rows.numel())
    got = run_head(h, x, ws, bs, rows, dl)
    ref = ref_head(h, x, ws, bs, rows, dl)
    close(got[0], ref[0])
    close(got[1], ref[1])
    close(got[2], ref[2])
    for a, b in zip(got[3] + got[4], ref[3] + ref[4]):
        close(a, b)
    outside = torch.ones(N, dtype=torch.bool)
    outside[rows.long()] = False
    assert (got[1][outside] == 0).all() and (got[2][outside] == 0).all()


@pytest.mark.parametrize("det", [0, 1])
def test_head_weight_gradients_are_bit_reproducible(det):
    L_ = _lib.lib()
    old = L_.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC)
    L_.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, det)
    try:
        N = 20000
        rows = np.sort(np.random.default_rng(0).choice(N, size=9000, replace=False))
        h, x, ws, bs, rows = head_case(N, 64, 3, rows)
        dl = torch.randn(rows.numel())
        a, b = run_head(h, x, ws, bs, rows, dl), run_head(h, x, ws, bs, rows, dl)
        for p, q in zip(a[1:3] + tuple(a[3] + a[4]), b[1:3] + tuple(b[3] + b[4])):
            assert torch.equal(p, q)
    finally:
        L_.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, old)


@pytest.mark.parametrize("pw", [1.0, 3.0])
def test_node_bce_matches_torch(pw):
    N = 5000
    rows = torch.as_tensor(np.sort(np.random.default_rng(2).choice(N, 1234, replace=False)), dtype=torch.int32)
    vuln = torch.as_tensor(random_vuln(N, 0.3, 5), dtype=torch.int32)
    logits = torch.randn(N) * 3
    S = torch.tensor([rows.numel()], dtype=torch.int32, device=DEV)
    rows_d = torch.zeros(N, dtype=torch.int32, device=DEV)
    rows_d[: rows.numel()] = rows.to(DEV)
    loss = torch.zeros(1, device=DEV)
    with torch.cuda.device(DEV):
        dl = E.node_bce(logits.to(DEV), vuln.to(DEV), rows_d, S, pw, loss)
    lg = logits[: rows.numel()].double().requires_grad_(True)
    ref = torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor([pw], dtype=torch.float64))(lg, vuln[rows.long()].double())
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    close(dl[: rows.numel()].cpu(), lg.grad, 1e-5)
    S.zero_()
    with torch.cuda.device(DEV):
        E.node_bce(logits.to(DEV), vuln.to(DEV), rows_d, S, pw, loss)
    assert torch.isnan(loss).all(), "a mean over no rows is NaN, as in torch"


# ---- the trainer -----------------------------------------------------------------------------------------------------------
def node_module(engine, factor=1.0, pw=None, seed=1):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, label_style="node", concat_all_absdf=True, engine=engine,
                               undersample_node_on_loss_factor=factor, positive_weight=pw).to(DEV)


def batches(n, seed=300, graphs=12, nodes=40, vuln_rate=0.5):
    return [synth.make_batch(graphs, nodes, seed=seed + i, variable=True, vuln_rate=vuln_rate) for i in range(n)]


def module_path(engine, factor, pw, bs, rows_per_step, lr=1e-3, wd=1e-2, max_norm=None):
    m = node_module(engine, factor, pw)
    opt = torch.optim.Adam(m.parameters(), lr=lr, weight_decay=wd)
    losses, norms = [], []
    for b, rows in zip(bs, rows_per_step):
        opt.zero_grad()
        out = m(b)
        label = m.get_label(b)
        idx = rows.long().to(DEV)
        loss = m.loss_fn(out[idx], label[idx])
        loss.backward()
        if max_norm is not None:
            norms.append(float(torch.nn.utils.clip_grad_norm_(m.parameters(), max_norm)))
        opt.step()
        losses.append(float(loss))
    return losses, [p.detach().clone() for p in m.parameters()], norms


def trainer_run(engine, factor, pw, bs, seed=0, **kw):
    m = node_module(engine, factor, pw)
    tr = D.FusedTrainer(m, lr=1e-3, weight_decay=1e-2, node_sample_seed=seed, **kw)
    losses, rows = [], []
    for b in bs:
        losses.append(float(tr.step(b if kw.get("use_cuda_graph") else b.to(DEV))))
        rows.append(tr.last_loss_rows().cpu())
    return losses, [p.detach().clone() for p in m.parameters()], rows, tr


def engines():
    return ["simt", "tcgen05"] if _lib.lib().call("ddfa_engine_available", 1) else ["simt"]


def nan_eq(a, b):
    return (a == b) or (a != a and b != b)


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("factor,pw", [(None, None), (1.0, None), (2.0, 3.0)])
@pytest.mark.parametrize("steps", [1, 20])
def test_trainer_matches_the_module_path(engine, factor, pw, steps):
    if engine not in engines():
        pytest.skip("tcgen05 engine not compiled in")
    bs = batches(steps)
    lt, pt, rows, _ = trainer_run(engine, factor, pw, bs)
    for b, r in zip(bs, rows):
        v = b.ndata["_VULN"]
        assert int((v[r.long()] != 0).sum()) == int((v != 0).sum())
        if factor is None:
            assert r.numel() == b.num_nodes()
        else:
            assert r.numel() == int((v != 0).sum()) + E.undersample_count(int((v != 0).sum()), factor)
    l1, p1, _ = module_path(engine, factor, pw, bs, rows)
    l2, p2, _ = module_path(engine, factor, pw, bs, rows)
    noise_l = max(abs(a - b) for a, b in zip(l1, l2))
    noise_p = max(float((a - b).abs().max()) for a, b in zip(p1, p2))
    dl = max(abs(a - b) for a, b in zip(lt, l1))
    dp = max(float((a - b).abs().max()) for a, b in zip(pt, p1))
    print(f"{engine} factor={factor} pw={pw} steps={steps}: |dloss| {dl:.2e} |dparam| {dp:.2e} (module path twice: {noise_l:.2e} / {noise_p:.2e})")
    assert dl <= 4 * noise_l + 2e-5 * max(1.0, max(abs(v) for v in l1))
    assert dp <= 4 * noise_p + (2e-5 if steps == 1 else 2e-4)


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_batch_without_vulnerable_nodes(engine):
    """Undersampling and no vulnerable node: S = 0, loss NaN, zero gradients, parameters moved by weight decay alone."""
    if engine not in engines():
        pytest.skip("tcgen05 engine not compiled in")
    b = synth.make_batch(8, 30, seed=5, vuln_rate=0.0)
    b.ndata["_VULN"].zero_()
    lt, pt, rows, _ = trainer_run(engine, 1.0, None, [b])
    assert rows[0].numel() == 0 and lt[0] != lt[0]
    lm, pm, _ = module_path(engine, 1.0, None, [b], rows)
    assert lm[0] != lm[0]
    for a, c in zip(pt, pm):
        assert (a - c).abs().max() <= 1e-7


def test_oversized_draw_raises_value_error():
    bs = batches(2, vuln_rate=0.6)
    m = node_module("simt", 500.0)
    tr = D.FusedTrainer(m)
    tr.step(bs[0].to(DEV))
    with pytest.raises(ValueError, match="more non-vulnerable"):
        tr.check_inputs()
    tr.check_inputs()                      # reported once
    tr.step(bs[0].to(DEV))
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="more non-vulnerable"):
        tr.step(bs[1].to(DEV))


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_eager_and_captured_agree_bit_for_bit(engine, deterministic):
    if engine not in engines():
        pytest.skip("tcgen05 engine not compiled in")
    bs = [synth.make_batch(12, 40, seed=900 + (i % 2), vuln_rate=0.5) for i in range(6)]     # one shape: captured after two steps
    le, pe, re_, _ = trainer_run(engine, 1.0, 2.0, bs)
    lc, pc, rc, tr = trainer_run(engine, 1.0, 2.0, bs, use_cuda_graph=True)
    assert any(st["graph"] is not None for slot in tr._stream_slots.values() for st in slot["sets"])
    assert all(torch.equal(a, b) for a, b in zip(re_, rc))
    assert all(nan_eq(a, b) for a, b in zip(le, lc)) and all(torch.equal(a, b) for a, b in zip(pe, pc))


def test_bucketed_stream_draws_the_exact_shape_rows():
    bs = batches(6, seed=40)
    _, _, r_exact, _ = trainer_run("simt", 1.0, None, bs, use_cuda_graph=True)
    _, _, r_bucket, tr = trainer_run("simt", 1.0, None, bs, use_cuda_graph=True, bucket_nodes=512, bucket_edges=2048)
    assert tr.num_bucket_shapes() >= 1
    assert all(torch.equal(a, b) for a, b in zip(r_exact, r_bucket))


def test_step_ids_equals_host_batches(deterministic):
    graphs = [synth.make_batch(1, 30, seed=600 + i, vuln_rate=0.3) for i in range(30)]
    arena = D.GraphArena.from_graphs(graphs, DEV)
    ids = [np.random.default_rng(i).integers(0, 30, 8) for i in range(5)]
    m1 = node_module("simt", 1.0)
    t1 = D.FusedTrainer(m1, use_cuda_graph=True)
    m2 = node_module("simt", 1.0)
    t2 = D.FusedTrainer(m2)
    for i in ids:
        a = float(t1.step_ids(arena, i))
        r1 = t1.last_loss_rows()
        b = float(t2.step(arena.batch(i)))
        assert nan_eq(a, b) and torch.equal(r1, t2.last_loss_rows())
    assert all(torch.equal(p, q) for p, q in zip(m1.parameters(), m2.parameters()))


def test_deterministic_runs_and_resume_are_bit_identical(deterministic):
    bs = batches(20, seed=77)
    la, pa, ra, _ = trainer_run("simt", 1.0, 2.0, bs, seed=3)
    lb, pb, rb, _ = trainer_run("simt", 1.0, 2.0, bs, seed=3)
    assert all(nan_eq(a, b) for a, b in zip(la, lb)) and all(torch.equal(a, b) for a, b in zip(pa, pb))
    # resume at step 10
    m = node_module("simt", 1.0, 2.0)
    tr = D.FusedTrainer(m, lr=1e-3, weight_decay=1e-2, node_sample_seed=3)
    for b in bs[:10]:
        tr.step(b.to(DEV))
    state, opt, draws = copy.deepcopy(m.state_dict()), tr.optimizer.state_dict(), tr.node_sample_draws
    assert draws == 10
    m2 = node_module("simt", 1.0, 2.0, seed=99)
    m2.load_state_dict(state)
    tr2 = D.FusedTrainer(m2, lr=1e-3, weight_decay=1e-2, node_sample_seed=3)
    tr2.optimizer.load_state_dict(opt)
    tr2.node_sample_draws = draws
    lr_ = [float(tr2.step(b.to(DEV))) for b in bs[10:]]
    assert all(nan_eq(a, b) for a, b in zip(lr_, la[10:]))
    assert all(torch.equal(a, b) for a, b in zip([p.detach() for p in m2.parameters()], pa))


def test_max_grad_norm_clips_like_clip_grad_norm():
    bs = batches(3, seed=12)
    lt, pt, rows, tr = trainer_run("simt", 1.0, None, bs, max_grad_norm=0.05)
    lm, pm, norms = module_path("simt", 1.0, None, bs, rows, max_norm=0.05)
    assert norms[-1] > 0.05, "the bound must bite"
    assert abs(float(tr.grad_norm) - norms[-1]) <= 1e-4 * norms[-1]
    dp = max(float((a - b).abs().max()) for a, b in zip(pt, pm))
    assert dp <= 2e-5, dp
