"""GPU: parameter groups and AdamW in the fused Adam kernels and FusedTrainer(param_groups=..., decoupled_weight_decay=...).

Checked: ddfa_adam_flat_groups with one coupled group is ddfa_adam_flat_hp / ddfa_adam_flat_guarded bit for bit, several groups
are ddfa_adam_flat_ranges per group and leave every element outside the ranges alone, decoupled groups follow
torch.optim.AdamW(foreach=False) on the device; the peer-memory grouped kernel (1, 2 and 4 ranks emulated on one device) is
the single-rank grouped kernel bit for bit.  The trainer with a decay / no-decay split under AdamW follows module.training_step +
torch.optim.AdamW on the same groups (both engines, both label styles); its step paths agree bit for bit; a group at lr = 0 stays
put, also in captured replays after a LambdaLR change; a checkpoint resumes bit-identically through torch.optim.AdamW; one
coupled group over everything gives the default trainer's bits with the guard, accumulation and frozen parameters; deterministic
runs repeat; and without the new arguments the step enqueues the kernels it always did."""
import contextlib
import copy
import gc
import os
import socket

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200._lib import lib, ptr_array
from deepdfa_b200.engine import _p, _stream_ptr
from deepdfa_b200.trainer import group_row

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
HP = [1e-3, 0.9, 0.999, 1e-8, 1e-2]


@contextlib.contextmanager
def det_mode(on=True):
    prev = os.environ.get("DDFA_DETERMINISTIC")
    os.environ["DDFA_DETERMINISTIC"] = "1" if on else "0"
    try:
        yield
    finally:
        if prev is None:
            os.environ.pop("DDFA_DETERMINISTIC")
        else:
            os.environ["DDFA_DETERMINISTIC"] = prev
        _lib.apply_deterministic_mode()


def table(rows):
    return torch.tensor([list(r) for r in rows], dtype=torch.float32, device=DEV)


def row(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, wd=1e-2, decoupled=False):
    return group_row(dict(lr=lr, betas=betas, eps=eps, weight_decay=wd, decoupled_weight_decay=decoupled))


def flat_groups(p, g, m, v, step, ranges, rows, gstate=None, skipped=None):
    rdev = torch.tensor(ranges, dtype=torch.int64, device=DEV).reshape(-1)
    tab = table(rows)
    lib().call("ddfa_adam_flat_groups", _p(p), _p(g), _p(m), _p(v), _p(step), p.numel(), _p(rdev), len(ranges), _p(tab), len(rows),
               _p(gstate) if gstate is not None else None, _p(skipped) if skipped is not None else None, _stream_ptr())
    torch.cuda.synchronize()       # rdev / tab are freed on return


# ---- 1. the flat kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("guarded", [False, True])
def test_one_coupled_group_is_the_single_group_kernel_bit_for_bit(guarded):
    torch.manual_seed(5)
    n = 64 * 97
    init = [torch.randn(n, device=DEV), torch.rand(n, device=DEV) * 0.1, torch.rand(n, device=DEV) * 0.01]
    a, b = [t.clone() for t in init], [t.clone() for t in init]
    sa, sb = (torch.full((1,), 2, dtype=torch.int32, device=DEV) for _ in range(2))
    hyper = torch.tensor(HP, device=DEV)
    gstate = torch.tensor([1.0, 0.37, 0.0, 0.0], device=DEV)
    for _ in range(4):
        g = torch.randn(n, device=DEV) * 0.01
        if guarded:
            lib().call("ddfa_adam_flat_guarded", _p(a[0]), _p(g), _p(a[1]), _p(a[2]), _p(sa), n, _p(hyper), _p(gstate), None, _stream_ptr())
        else:
            lib().call("ddfa_adam_flat_hp", _p(a[0]), _p(g), _p(a[1]), _p(a[2]), _p(sa), n, _p(hyper), _stream_ptr())
        flat_groups(b[0], g, b[1], b[2], sb, [(0, n, 0)], [row(*HP[:1], betas=HP[1:3], eps=HP[3], wd=HP[4])],
                    gstate=gstate if guarded else None)
    torch.cuda.synchronize()
    assert int(sa) == int(sb) == 6
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_groups_are_the_ranged_kernel_per_group_and_leave_the_rest_alone():
    torch.manual_seed(6)
    n = 64 * 97
    ranges = [(0, 128, 1), (128, 512, 0), (1024, 2048, 2), (2048, 2112, 1), (4096, n, 0)]
    hps = [[1e-3, 0.9, 0.999, 1e-8, 1e-2], [5e-3, 0.8, 0.99, 1e-6, 0.0], [0.0, 0.9, 0.999, 1e-8, 0.0]]
    rows = [row(h[0], (h[1], h[2]), h[3], h[4]) for h in hps]
    init = [torch.randn(n, device=DEV), torch.rand(n, device=DEV) * 0.1, torch.rand(n, device=DEV) * 0.01]
    grouped = [t.clone() for t in init]
    per = [[t.clone() for t in init] for _ in hps]
    sg = torch.zeros(1, dtype=torch.int32, device=DEV)
    sp = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in hps]
    skipped = torch.zeros(1, dtype=torch.int32, device=DEV)
    gstate = torch.tensor([1.0, 1.0, 0.0, 0.0], device=DEV)
    for _ in range(3):
        g = torch.randn(n, device=DEV) * 0.01
        flat_groups(grouped[0], g, grouped[1], grouped[2], sg, ranges, rows, gstate=gstate, skipped=skipped)
        for k, h in enumerate(hps):
            rk = torch.tensor([(a, b) for a, b, gi in ranges if gi == k], dtype=torch.int64, device=DEV).reshape(-1)
            lib().call("ddfa_adam_flat_ranges", _p(per[k][0]), _p(g), _p(per[k][1]), _p(per[k][2]), _p(sp[k]), n, _p(rk), rk.numel() // 2,
                       _p(torch.tensor(h, device=DEV)), _p(gstate), _p(skipped), _stream_ptr())
            torch.cuda.synchronize()
    assert int(sg) == 3 and int(skipped) == 0
    outside = torch.ones(n, dtype=torch.bool, device=DEV)
    for a, b, k in ranges:
        outside[a:b] = False
        for x, y in zip(grouped, per[k]):
            assert torch.equal(x[a:b], y[a:b]), (a, b, k)
    for x, x0 in zip(grouped, init):
        assert torch.equal(x[outside], x0[outside])          # sentinels: bit-unchanged
    assert torch.equal(grouped[0][1024:2048], init[0][1024:2048])     # lr = 0, wd = 0: the parameters stay put


def test_decoupled_groups_follow_torch_adamw():
    """Two AdamW groups and one coupled group over one buffer, 40 steps, against torch.optim.AdamW / Adam(foreach=False) on
    the same device; the worst difference is reported in ulps."""
    torch.manual_seed(7)
    segs = [(0, 1024), (1024, 3072), (3072, 4096)]
    cfg = [dict(lr=1e-3, weight_decay=0.1, decoupled_weight_decay=True), dict(lr=3e-3, weight_decay=0.0, decoupled_weight_decay=True),
           dict(lr=2e-3, weight_decay=1e-2, decoupled_weight_decay=False)]
    n = segs[-1][1]
    p0 = torch.randn(n, device=DEV)
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    refs = [torch.nn.Parameter(p0[a:b].clone()) for a, b in segs]
    opt = torch.optim.AdamW([dict(params=[r], **c) for r, c in zip(refs, cfg)], foreach=False)
    rows = [group_row(dict(opt.param_groups[k])) for k in range(3)]
    assert rows[0][5] == 1.0 and rows[2][5] == 0.0
    for _ in range(40):
        g = torch.randn(n, device=DEV) * 0.05
        flat_groups(p, g, m, v, step, [(a, b, k) for k, (a, b) in enumerate(segs)], rows)
        for r, (a, b) in zip(refs, segs):
            r.grad = g[a:b].clone()
        opt.step()
    ref = torch.cat([r.detach() for r in refs])
    diff = float((p - ref).abs().max())
    same_sign = (p.sign() == ref.sign()) & (ref.abs() > 1e-3)
    ulps = int((p.view(torch.int32).long() - ref.view(torch.int32).long()).abs()[same_sign].max())
    moved = float((ref - p0).abs().max())
    print(f"AdamW groups vs torch.optim.AdamW(foreach=False), 40 steps: max |dp| {diff:.2e}, worst {ulps} ulps (moved {moved:.2e})")
    assert moved > 1e-2 and diff < 2e-6


# ---- 2. the peer-memory kernel, ranks emulated on one device ------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("guarded", [False, True])
def test_p2p_groups_are_the_flat_grouped_kernel_bit_for_bit(world, guarded):
    torch.manual_seed(world + 10 * guarded)
    n = 64 * 97
    ranges = [(0, 256, 1), (256, 1024, 0), (2048, 4096, 2), (4096, n, 1)]       # [1024, 2048) is outside: sentinels
    rows = [row(1e-3, wd=0.1, decoupled=True), row(2e-3, wd=0.0, decoupled=True), row(1e-3, wd=1e-2)]
    rdev = torch.tensor(ranges, dtype=torch.int64, device=DEV).reshape(-1)
    tab = table(rows)
    p0 = torch.randn(n, device=DEV)
    params = [p0.clone() for _ in range(world)]
    grads = [torch.zeros(n + 64, device=DEV) for _ in range(world)]
    flags = [torch.zeros(128, dtype=torch.int32, device=DEV) for _ in range(world)]
    m = [torch.zeros(n, device=DEV) for _ in range(world)]
    v = [torch.zeros(n, device=DEV) for _ in range(world)]
    step = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)]
    ticket = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)]
    gws = [torch.zeros(lib().call("ddfa_p2p_guard_state_bytes"), dtype=torch.uint8, device=DEV) for _ in range(world)]
    gst = [torch.zeros(4, device=DEV) for _ in range(world)]
    loss_out = [torch.zeros(1, device=DEV) for _ in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    fp, fm, fv, fs = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    gflat = torch.tensor([0.0, 1.0, 0.0, 0.0], device=DEV)          # coef 1: the p2p kernel measures without a bound
    pp, pg, pf = ptr_array([_p(t) for t in params]), ptr_array([_p(t) for t in grads]), ptr_array([_p(t) for t in flags])
    for it in range(4):
        gs = [torch.randn(n, device=DEV) * 0.1 for _ in range(world)]
        for r in range(world):
            grads[r][:n].copy_(gs[r])
            grads[r][n] = float(r + 1)
        torch.cuda.synchronize()
        for r in range(world):
            head = (pp, pg, pf, r, world, _p(m[r]), _p(v[r]), _p(step[r]), n, n, _p(loss_out[r]))
            if guarded:
                lib().call("ddfa_allreduce_adam_p2p_groups_guarded", *head, _p(rdev), len(ranges), _p(tab), len(rows), None, _p(gst[r]),
                           None, _p(gws[r]), streams[r].cuda_stream)
            else:
                lib().call("ddfa_allreduce_adam_p2p_groups", *head, _p(ticket[r]), _p(rdev), len(ranges), _p(tab), len(rows),
                           streams[r].cuda_stream)
        torch.cuda.synchronize()
        red = torch.zeros(n, device=DEV)
        for gr in gs:
            red = red + gr                                     # the kernel's rank-order fp32 sum
        flat_groups(fp, red, fm, fv, fs, ranges, rows, gstate=gflat if guarded else None)
        for r in range(world):
            assert torch.equal(params[r], fp), (it, r)
            assert int(step[r]) == it + 1
            if guarded:
                assert float(gst[r][1]) == 1.0
                assert abs(float(gst[r][0]) - float(red.double().norm())) <= 1e-5 * float(red.double().norm())
    assert torch.equal(fp[1024:2048], p0[1024:2048])
    from deepdfa_b200.trainer import owned_range
    for r in range(world):                                   # each rank holds the moments of its slice
        lo, hi = owned_range(n, r, world)
        assert torch.equal(m[r][lo:hi], fm[lo:hi]) and torch.equal(v[r][lo:hi], fv[lo:hi])


# ---- 3. the trainer against the module path + torch.optim.AdamW ---------------------------------------------------------
def module(engine="tcgen05", style="graph", seed=1, factor=None, device=DEV):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, label_style=style, concat_all_absdf=True, positive_weight=2.0,
                               undersample_node_on_loss_factor=factor, engine=engine).to(device)


def decay_split(m, wd=0.1, lr_decay=1e-3, lr_no_decay=2e-3):
    """linevul_main.py's grouping: biases without weight decay; here also a learning rate per group."""
    decay = [p for n, p in m.named_parameters() if "bias" not in n]
    no_decay = [p for n, p in m.named_parameters() if "bias" in n]
    return [{"params": decay, "weight_decay": wd, "lr": lr_decay}, {"params": no_decay, "weight_decay": 0.0, "lr": lr_no_decay}]


def graph_batches(n, seed=700, graphs=16, nodes=40):
    return [synth.make_batch(graphs, nodes, seed=seed + i, variable=True, vuln_rate=0.3) for i in range(n)]


def adamw_trainer(m, **kw):
    return D.FusedTrainer(m, param_groups=decay_split(m), decoupled_weight_decay=True, **kw)


def torch_adamw_run(engine, style, factor, bs, rows):
    m = module(engine, style, seed=2, factor=factor)
    opt = torch.optim.AdamW(decay_split(m))
    losses = []
    for i, b in enumerate(bs):
        opt.zero_grad()
        b = b.to(DEV)
        if style == "node":
            idx = rows[i].long().to(DEV)
            loss = m.loss_fn(m(b)[idx], m.get_label(b)[idx])
        else:
            loss = m.training_step((b, {}), 0)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return losses, m, opt


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("style", ["graph", "node"])
def test_adamw_decay_split_follows_torch_adamw(engine, style):
    """Tolerances as in the frozen-parameter and node-style trainer tests, plus 4x the module path's own run-to-run spread.
    pooling.gate_nn.bias has a zero gradient in exact arithmetic (the readout softmax is shift-invariant); in the no-decay group
    Adam steps on its rounding noise on either side, so it is held to Adam's step bound instead."""
    factor = 1.0 if style == "node" else None
    bs = graph_batches(16, seed=300)
    mf = module(engine, style, seed=2, factor=factor)
    tr = adamw_trainer(mf)
    assert [name for name, _ in tr._update] == ["ddfa_adam_flat_groups"]
    lf, rows = [], []
    for b in bs:
        lf.append(float(tr.step(b.to(DEV))))
        if style == "node":
            rows.append(tr.last_loss_rows().cpu())
    lr_, mr, opt = torch_adamw_run(engine, style, factor, bs, rows)
    _, mr2, _ = torch_adamw_run(engine, style, factor, bs, rows)
    noise = max(float((p - q).abs().max()) for p, q in zip(mr.parameters(), mr2.parameters()))
    zero_grad = {"pooling.gate_nn.bias"}
    diffs = {n: float((p - q).abs().max()) for (n, p), q in zip(mf.named_parameters(), mr.parameters())}
    dl = max(abs(a - b) / max(1.0, abs(b)) for a, b in zip(lf, lr_))
    dp = max(d for n, d in diffs.items() if n not in zero_grad)
    print(f"{style} {engine} AdamW decay split: max rel |dloss| {dl:.2e}, max |dparam| {dp:.2e} (torch twice: {noise:.2e}), "
          f"gate bias {diffs.get('pooling.gate_nn.bias', 0.0):.2e}")
    assert dl < (2e-5 if engine == "simt" else 2e-3)
    assert dp <= 4 * noise + ((1e-4 if style == "graph" else 2e-4) if engine == "simt" else 1e-3)
    for n in zero_grad & set(diffs):
        assert diffs[n] <= 2 * 2e-3 * len(bs)                   # two Adam trajectories of at most ~lr per step each
    sd_f, sd_t = tr.optimizer.state_dict(), opt.state_dict()
    assert sd_f["param_groups"] == sd_t["param_groups"]
    assert sorted(sd_f["state"]) == sorted(sd_t["state"])


def run_state(m, tr):
    torch.cuda.synchronize()
    return [p.detach().clone() for p in m.parameters()] + [tr.exp_avg.clone(), tr.exp_avg_sq.clone(), tr.step_count.clone()]


def assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (i, float((x.double() - y.double()).abs().max()))


def test_step_paths_are_bit_identical():
    bs = [synth.make_batch(16, 40, seed=40 + i % 2, vuln_rate=0.3) for i in range(6)]
    dev_bs = [b.to(DEV) for b in bs]
    with det_mode():
        out = {}
        for path in ("eager", "resident", "host"):
            m = module(seed=3)
            tr = adamw_trainer(m, use_cuda_graph=path != "eager")
            losses = [float(tr.step(b if path == "host" else d)) for b, d in zip(bs, dev_bs)]
            out[path] = (losses, run_state(m, tr))
            if path == "resident":
                assert len(tr._graphs) >= 1
            if path == "host":
                assert all(st["graph"] is not None for s in tr._stream_slots.values() for st in s["sets"])
        for path in ("resident", "host"):
            assert out[path][0] == out["eager"][0], path
            assert_same(out[path][1], out["eager"][1])
        graphs = [synth.make_batch(1, 30, seed=600 + i, vuln_rate=0.3) for i in range(30)]
        arena = D.GraphArena.from_graphs(graphs, DEV)
        ids = [np.random.default_rng(i % 2).integers(0, 30, 8) for i in range(5)]
        m1, m2 = module(seed=4), module(seed=4)
        t1, t2 = adamw_trainer(m1, use_cuda_graph=True), adamw_trainer(m2)
        for i in ids:
            assert float(t1.step_ids(arena, i)) == float(t2.step(arena.batch(i)))
        assert_same(run_state(m1, t1), run_state(m2, t2))


@pytest.mark.parametrize("path", ["eager", "resident", "host", "bucketed", "arena"])
def test_one_coupled_group_over_everything_is_the_default_trainer_on_every_path(path):
    """The grouped entry points on every step path: one coupled group with the trainer's hyperparameters gives the default
    trainer's bits (ddfa_adam_flat_groups is ddfa_adam_flat_hp there)."""
    bs = graph_batches(6, seed=410, graphs=12, nodes=30)
    kw = {"eager": {}, "resident": dict(use_cuda_graph=True), "host": dict(use_cuda_graph=True),
          "bucketed": dict(use_cuda_graph=True, bucket_nodes=64, bucket_edges=256, bucket_min_pad_nodes=8, max_graph_shapes=16),
          "arena": dict(use_cuda_graph=True)}[path]
    arena = D.GraphArena.from_graphs([synth.make_batch(1, 30, seed=600 + i, vuln_rate=0.3) for i in range(30)], DEV)
    ids = [np.random.default_rng(i % 3).integers(0, 30, 8) for i in range(6)]
    dev_bs = [b.to(DEV) for b in bs]
    runs = []
    with det_mode():
        for grouped in (False, True):
            m = module(seed=5)
            tr = D.FusedTrainer(m, param_groups=[{"params": list(m.parameters())}] if grouped else None, **kw)
            assert tr._update[-1][0] == ("ddfa_adam_flat_groups" if grouped else "ddfa_adam_flat_hp")
            for i in range(12):
                if path == "arena":
                    tr.step_ids(arena, ids[i % 6])
                else:
                    tr.step(dev_bs[i % 6] if path in ("eager", "resident") else bs[i % 6])
            runs.append(run_state(m, tr))
    assert_same(runs[0], runs[1])


def test_zero_lr_group_stays_put_in_captured_replays_after_a_scheduler_change():
    b = graph_batches(1, seed=500)[0]          # one shape: eager, two captures, then replays only
    m = module(seed=6)
    m0 = [p.detach().clone() for p in m.parameters()]
    names = [n for n, _ in m.named_parameters()]
    head = [p for n, p in m.named_parameters() if n.startswith("output_layer.")]
    ggnn = [p for n, p in m.named_parameters() if n.startswith("ggnn.")]
    rest = [p for n, p in m.named_parameters() if not n.startswith(("output_layer.", "ggnn."))]
    groups = [{"params": head, "lr": 0.0, "weight_decay": 0.0}, {"params": ggnn, "weight_decay": 0.1}, {"params": rest}]
    tr = D.FusedTrainer(m, param_groups=groups, decoupled_weight_decay=True, use_cuda_graph=True)
    sched = torch.optim.lr_scheduler.LambdaLR(tr.optimizer, [lambda s: 1.0, lambda s: 1.0 if s < 4 else 0.0, lambda s: 0.5 ** s])
    where = {n: i for i, n in enumerate(names)}
    ggnn_ids = [i for i, n in enumerate(names) if n.startswith("ggnn.")]
    at_change = None
    for i in range(10):
        tr.step(b)
        sched.step()
        if i == 3:
            torch.cuda.synchronize()
            at_change = [list(m.parameters())[k].detach().clone() for k in ggnn_ids]
            graphs_before = [id(st["graph"]) for s in tr._stream_slots.values() for st in s["sets"]]
            assert all(st["graph"] is not None for s in tr._stream_slots.values() for st in s["sets"])
    torch.cuda.synchronize()
    ps = list(m.parameters())
    for n, p in m.named_parameters():
        if n.startswith("output_layer."):
            assert torch.equal(p.detach(), m0[where[n]]), n            # lr = 0 from the start
        elif not n.startswith("ggnn."):
            assert not torch.equal(p.detach(), m0[where[n]]), n        # the third group moved
    for k, before in zip(ggnn_ids, at_change):
        assert not torch.equal(before, m0[k])                         # moved until the change ...
        assert torch.equal(ps[k].detach(), before)                    # ... then stayed put in the replays
    assert [id(st["graph"]) for s in tr._stream_slots.values() for st in s["sets"]] == graphs_before
    assert int(tr.step_count) == 10
    assert float(tr.hyper[1, 0]) == 0.0 and float(tr.hyper[1, 6]) == 1.0


def test_checkpoint_round_trip_through_torch_adamw_resumes_bit_identically():
    bs = [b.to(DEV) for b in graph_batches(8, seed=800)]
    with det_mode():
        ma = module("simt", seed=7)
        ta = adamw_trainer(ma)
        for b in bs[:4]:
            ta.step(b)
        sd = copy.deepcopy(ta.optimizer.state_dict())
        # through torch: a torch.optim.AdamW on the same groups loads it and saves it again
        mt = module("simt", seed=99)
        mt.load_state_dict(copy.deepcopy(ma.state_dict()))
        opt = torch.optim.AdamW(decay_split(mt))
        opt.load_state_dict(sd)
        sd2 = copy.deepcopy(opt.state_dict())
        assert sd2["param_groups"] == sd["param_groups"] and all(g["decoupled_weight_decay"] for g in sd2["param_groups"])
        mb = module("simt", seed=99)
        mb.load_state_dict(copy.deepcopy(ma.state_dict()))
        tb = adamw_trainer(mb)
        tb.optimizer.load_state_dict(sd2)
        assert int(tb.step_count) == 4
        for b in bs[4:]:
            ta.step(b)
            tb.step(b)
        assert_same(run_state(ma, ta), run_state(mb, tb))
        # a different group structure is refused, as torch refuses it
        bad = copy.deepcopy(sd2)
        bad["param_groups"].append(dict(bad["param_groups"][0], params=[]))
        with pytest.raises(ValueError):
            tb.optimizer.load_state_dict(bad)


@pytest.mark.parametrize("case", ["guard", "accumulate", "frozen_mix"])
def test_one_coupled_group_keeps_the_single_group_rules(case):
    """The guard (clipping and a skipped non-finite step), k = 2 accumulation and a partly frozen model with a frozen tensor
    listed in the group: one coupled group over the parameters gives the default trainer's bits."""
    bs = [b.to(DEV) for b in graph_batches(6, seed=900)]
    kw = {"guard": dict(max_grad_norm=0.05, skip_nonfinite=True), "accumulate": dict(accumulate_grad_batches=2),
          "frozen_mix": dict(max_grad_norm=1.0)}[case]
    runs = []
    with det_mode():
        for grouped in (False, True):
            m = module(seed=8)
            if case == "frozen_mix":
                for n, p in m.named_parameters():
                    if "embedding" in n or n == "ggnn.gru.weight_hh":
                        p.requires_grad_(False)
            tr = D.FusedTrainer(m, param_groups=[{"params": list(m.parameters())}] if grouped else None, **kw)
            for i, b in enumerate(bs):
                if case == "guard" and i == 3:
                    t = m.param_list()[0]
                    keep = t.data.clone()
                    t.data.fill_(float("nan"))
                    tr.step(b)
                    torch.cuda.synchronize()
                    t.data.copy_(keep)
                else:
                    tr.step(b)
            runs.append(run_state(m, tr) + ([tr._skipped.clone(), tr._gstate.clone()] if "max_grad_norm" in kw else []))
            if case == "guard":
                assert tr.skipped_steps == 1
    assert_same(runs[0], runs[1])


@pytest.mark.parametrize("style", ["graph", "node"])
def test_deterministic_adamw_runs_are_bit_identical(style):
    bs = [b.to(DEV) for b in graph_batches(6, seed=77)]
    runs = []
    with det_mode():
        for _ in range(2):
            m = module(style=style, factor=1.0 if style == "node" else None)
            tr = adamw_trainer(m, node_sample_seed=3)
            losses = [float(tr.step(b)) for b in bs]
            runs.append((losses, run_state(m, tr)))
    assert runs[0][0] == runs[1][0]
    assert_same(runs[0][1], runs[1][1])


def cuda_kernels(fn):
    """The names of the device activities ``fn`` enqueues (sorted) and the library's launch count over it.  Work enqueued
    before the call finishes first, so none of it is recorded in the window, and the garbage earlier tests left is collected
    first, so none of it is released inside the window."""
    from torch.profiler import ProfilerActivity, profile
    gc.collect()
    torch.cuda.synchronize()
    n0 = lib().call("ddfa_launch_count")
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = sorted(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return names, lib().call("ddfa_launch_count") - n0


@pytest.mark.parametrize("style", ["graph", "node"])
def test_without_the_arguments_the_step_enqueues_what_it_did(style):
    b = graph_batches(1)[0].to(DEV)
    seen = []
    for kw in ({}, {"param_groups": None, "decoupled_weight_decay": False}, {"decoupled_weight_decay": True}):
        tr = D.FusedTrainer(module(style=style, factor=1.0), **kw)
        tr.step(b)                                            # warm-up: workspace growth
        tr.step(b)                                            # capture (its gc.collect / empty_cache stay out of the window)
        seen.append(cuda_kernels(lambda: tr.step(b)))         # the step every later step replays
    assert seen[0][1] > 0 and seen[0] == seen[1]
    assert any("adam_flat_kernel" in n for n in seen[0][0]) and not any("adam_flat_groups" in n for n in seen[0][0])
    # AdamW swaps the one update kernel for its grouped form and launches no more
    assert seen[2][1] == seen[0][1] and any("adam_flat_groups_kernel" in n for n in seen[2][0])


# ---- 4. two ranks ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, exchange, q):
    import torch.distributed as dist
    from deepdfa_b200.batched_graph import split_batch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2", DDFA_DETERMINISTIC="1")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    try:
        full = [synth.make_batch(64, 60, seed=900 + i, variable=True, vuln_rate=0.3) for i in range(4)]
        m = module(seed=7, device=dev)
        tr = D.FusedTrainer(m, distributed=True, exchange=exchange, param_groups=decay_split(m), decoupled_weight_decay=True,
                            max_grad_norm=1.0)
        for i in range(6):
            tr.step(split_batch(full[i % 4], 2)[rank].to(dev), global_batch=64)
        sd = tr.optimizer.state_dict()           # collective under p2p
        m1 = module(seed=7, device=dev)
        t1 = D.FusedTrainer(m1, distributed=False, param_groups=decay_split(m1), decoupled_weight_decay=True, max_grad_norm=1.0)
        for i in range(6):
            t1.step(full[i % 4].to(dev), global_batch=64)
        torch.cuda.synchronize()
        dp = max(float((p.data - r.data).abs().max()) for p, r in zip(m.param_list(), m1.param_list()))
        q.put((rank, (dp, tr.exchange, [name for name, _ in tr._update], sorted(sd["state"]) == sorted(t1.optimizer.state_dict()["state"]))))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_two_ranks_with_adamw_groups_match_one_rank(exchange):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, exchange, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(2):
            rank, out = q.get(timeout=600)
            res[rank] = out
    finally:
        for p in procs:
            p.join(timeout=120)
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(timeout=30)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    want = {"nccl": ["ddfa_grad_norm", "ddfa_adam_flat_groups"], "p2p": ["ddfa_allreduce_adam_p2p_groups_guarded"]}[exchange]
    for r in (0, 1):
        assert not isinstance(res[r], str), res[r]
        dp, used, calls, same_keys = res[r]
        assert used == exchange and calls == want and same_keys
        assert dp <= 1e-3, dp
