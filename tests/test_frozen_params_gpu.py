"""GPU: FusedTrainer with frozen parameters (requires_grad=False), e.g. the head refitted over a frozen graph encoder.

Checked: ddfa_adam_flat_ranges against ddfa_adam_flat_hp / ddfa_adam_flat_guarded (bit-identical inside the ranges, untouched
outside); the gate-only readout backward and the node head backward without input gradients against their full calls; the
trainer against module.training_step + torch.optim.Adam(model.parameters()) with the encoder, the tables, one GRU tensor or the
head frozen; the captured, bucketed and arena step paths against the eager step; clipping, NaN skipping, deterministic runs,
the optimizer state in torch's format, the error rules, two ranks, and the step's peak memory at C1."""
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
from deepdfa_b200 import engine as E
from deepdfa_b200._lib import lib
from deepdfa_b200.engine import _p, _stream_ptr
from deepdfa_b200.module import _ENGINES

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


def module(engine="tcgen05", style="graph", seed=1, steps=4, factor=None, device=DEV, graphs_hidden=32):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, graphs_hidden, steps, 2, label_style=style, concat_all_absdf=True, positive_weight=2.0,
                               undersample_node_on_loss_factor=factor, engine=engine).to(device)


def freeze(m, what):
    """encoder: main_cli.py:136-144's split (everything but output_layer.* / pooling.*); tables: the embedding tables; gru_whh:
    ggnn.gru.weight_hh alone; head: output_layer.* and pooling.*."""
    for name, p in m.named_parameters():
        head = name.startswith(("output_layer.", "pooling."))
        if {"encoder": not head, "tables": "embedding" in name, "gru_whh": name == "ggnn.gru.weight_hh", "head": head}[what]:
            p.requires_grad_(False)
    assert any(not p.requires_grad for p in m.parameters())
    return m


def graph_batches(n, seed=700, graphs=16, nodes=40):
    return [synth.make_batch(graphs, nodes, seed=seed + i, variable=True, vuln_rate=0.3) for i in range(n)]


# ---- 1. Adam over ranges -----------------------------------------------------------------------------------------------
RANGES = {"one": [(64, 640)], "two": [(0, 128), (512, 1024)], "many": [(128 * i, 128 * i + 64) for i in range(48)],
          "to_end": [(256, 320), (4096, 64 * 97)]}


@pytest.mark.parametrize("which", sorted(RANGES))
@pytest.mark.parametrize("guarded", [False, True])
def test_adam_flat_ranges_is_the_flat_update_on_the_range_elements(which, guarded):
    torch.manual_seed(3)
    n = 64 * 97
    ranges = RANGES[which]
    inside = torch.zeros(n, dtype=torch.bool)
    for a, b in ranges:
        inside[a:b] = True
    init = [torch.randn(n, device=DEV), torch.rand(n, device=DEV) * 0.1, torch.rand(n, device=DEV) * 0.01]
    full, part = [t.clone() for t in init], [t.clone() for t in init]
    sf, sp = (torch.full((1,), 4, dtype=torch.int32, device=DEV) for _ in range(2))
    hyper = torch.tensor(HP, device=DEV)
    rdev = torch.tensor(ranges, dtype=torch.int64, device=DEV).reshape(-1)
    gstate = torch.tensor([1.0, 0.37, 0.0, 0.0], device=DEV)          # [norm, coef, nonfinite]: a clipping step
    for _ in range(3):
        g = torch.randn(n, device=DEV) * 0.01
        if guarded:
            lib().call("ddfa_adam_flat_guarded", _p(full[0]), _p(g), _p(full[1]), _p(full[2]), _p(sf), n, _p(hyper), _p(gstate), None,
                       _stream_ptr())
        else:
            lib().call("ddfa_adam_flat_hp", _p(full[0]), _p(g), _p(full[1]), _p(full[2]), _p(sf), n, _p(hyper), _stream_ptr())
        lib().call("ddfa_adam_flat_ranges", _p(part[0]), _p(g), _p(part[1]), _p(part[2]), _p(sp), n, _p(rdev), len(ranges),
                   _p(hyper), _p(gstate) if guarded else None, None, _stream_ptr())
    torch.cuda.synchronize()
    assert int(sp) == int(sf) == 7
    m = inside.to(DEV)
    for f, p, i0 in zip(full, part, init):
        assert torch.equal(f[m], p[m])
        assert torch.equal(p[~m], i0[~m])


def test_adam_flat_ranges_skips_a_nonfinite_step():
    n = 1024
    p, m, v = torch.randn(n, device=DEV), torch.rand(n, device=DEV), torch.rand(n, device=DEV)
    step, skipped = torch.full((1,), 3, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    before = [t.clone() for t in (p, m, v, step)]
    rdev = torch.tensor([0, 512], dtype=torch.int64, device=DEV)
    gstate = torch.tensor([float("nan"), float("nan"), 1.0, 0.0], device=DEV)
    g = torch.randn(n, device=DEV)
    lib().call("ddfa_adam_flat_ranges", _p(p), _p(g), _p(m), _p(v), _p(step), n, _p(rdev), 1, _p(torch.tensor(HP, device=DEV)),
               _p(gstate), _p(skipped), _stream_ptr())
    torch.cuda.synchronize()
    assert int(skipped) == 1
    assert all(torch.equal(a, b) for a, b in zip(before, (p, m, v, step)))


# ---- 2. the pruned backward kernels ------------------------------------------------------------------------------------
def _close(a, b, rel=1e-4):
    return float((a - b).abs().max()) <= rel * max(1e-6, float(b.abs().max()))


@pytest.mark.parametrize("size", ["c1", "one_node"])
@pytest.mark.parametrize("det", [True, False])
def test_gate_only_readout_backward_matches_the_full_call(size, det):
    b = synth.make_batch(1024, 150, seed=5) if size == "c1" else synth.make_batch(sizes=[1], seed=5)
    m = module(steps=2, graphs_hidden=32)
    with det_mode(det):
        g, dg, idx = m._prepare(b.to(DEV))
        params = E.ParamPack.from_flat_list([p.detach() for p in m.param_list()], len(m._tables()), len(m._mlp_linears()))
        pooled, _, saved = E.forward(params, dg, idx, 2, training=True, engine=_ENGINES[m.engine])
        B, Dm = dg.batch_size, saved.D
        N = dg.num_nodes
        dpooled = torch.randn(B, 2 * Dm, device=DEV)
        ws_bytes = lib().call("ddfa_readout_bwd_workspace_bytes", B, Dm)
        ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=DEV)
        out = {}
        for form in ("full", "gate"):
            dw, db = torch.zeros(2 * Dm, device=DEV), torch.zeros(1, device=DEV)
            dh = torch.zeros(N, Dm, device=DEV) if form == "full" else None
            dx = torch.zeros(N, Dm, device=DEV) if form == "full" else None
            lib().call("ddfa_readout_bwd_ws", _p(dpooled), _p(saved.pooled), _p(saved.h[saved.T]), _p(saved.x), _p(dg.graph_ptr), B, Dm,
                       _p(params.w_gate), _p(saved.gate_logit), _p(saved.seg_max), _p(saved.seg_sum), _p(dh), _p(dx), _p(dw), _p(db),
                       _p(ws), ws_bytes, _stream_ptr())
            out[form] = (dw, db)
        torch.cuda.synchronize()
    for a, c in zip(out["full"], out["gate"]):
        assert torch.equal(a, c) if det else _close(c, a)
        assert float(a.abs().max()) > 0 or size == "one_node"      # softmax over one node: the gate gradient is exactly zero


@pytest.mark.parametrize("size", ["c1", "one_node"])
@pytest.mark.parametrize("det", [True, False])
def test_node_head_backward_without_input_grads_matches_the_full_call(size, det):
    b = synth.make_batch(1024, 150, seed=6) if size == "c1" else synth.make_batch(sizes=[1], seed=6)
    m = module(style="node", steps=2)
    with det_mode(det):
        g, dg, idx = m._prepare(b.to(DEV))
        params = E.ParamPack.from_flat_list([p.detach() for p in m.param_list()], len(m._tables()), len(m._mlp_linears()))
        x, h_T, _ = E.forward(params, dg, idx, 2, training=True, engine=_ENGINES[m.engine], head=False)
        N = x.shape[0]
        rows = torch.arange(N, dtype=torch.int32, device=DEV)
        S = torch.full((1,), N, dtype=torch.int32, device=DEV)
        _, act = E.node_head_fwd(params, x, h_T, rows, S)
        dlogits = torch.randn(N, device=DEV)
        out = {}
        for ig in (True, False):
            grads = params.zeros_like()
            E.node_head_bwd(params, grads, dlogits, x, h_T, rows, S, act, input_grads=ig)
            out[ig] = [t.clone() for t in grads.mlp_w + grads.mlp_b]
        torch.cuda.synchronize()
    for a, c in zip(out[True], out[False]):
        assert torch.equal(a, c)                 # fixed-order reductions in both modes


# ---- 3. the trainer against the module path + torch.optim.Adam ----------------------------------------------------------
def reference_graph(engine, what, bs, seed=2, max_norm=None):
    m = freeze(module(engine, seed=seed), what)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-2)
    losses, norms = [], []
    for b in bs:
        opt.zero_grad()
        loss = m.training_step((b.to(DEV), {}), 0)
        loss.backward()
        if max_norm is not None:
            norms.append(float(torch.nn.utils.clip_grad_norm_(m.parameters(), max_norm)))
        opt.step()
        losses.append(float(loss))
    return losses, m, opt, norms


def fused_graph(engine, what, bs, seed=2, **kw):
    m = freeze(module(engine, seed=seed), what)
    tr = D.FusedTrainer(m, lr=1e-3, weight_decay=1e-2, **kw)
    losses = [float(tr.step(b if kw.get("use_cuda_graph") else b.to(DEV))) for b in bs]
    return losses, m, tr


def assert_frozen_unchanged(m, seed, engine, what, style="graph", factor=None):
    init = freeze(module(engine, style=style, seed=seed, factor=factor), what)
    for p, q in zip(m.parameters(), init.parameters()):
        if not q.requires_grad:
            assert torch.equal(p.detach(), q.detach())


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("what", ["encoder", "tables", "gru_whh", "head"])
def test_graph_style_follows_torch_adam(engine, what):
    bs = graph_batches(20)
    lr_, mr, _, _ = reference_graph(engine, what, bs)
    lf, mf, tr = fused_graph(engine, what, bs)
    assert tr._grad_ggnn == (what != "encoder") and tr._grad_tables == (what not in ("encoder", "tables"))
    assert_frozen_unchanged(mf, 2, engine, what)
    assert_frozen_unchanged(mr, 2, engine, what)
    dl = max(abs(a - b) / max(1.0, abs(b)) for a, b in zip(lf, lr_))
    dp = max(float((p - q).abs().max()) for p, q in zip(mf.parameters(), mr.parameters()))
    print(f"graph {engine} frozen={what}: max rel |dloss| {dl:.2e}, max |dparam| {dp:.2e}")
    assert dl < (2e-5 if engine == "simt" else 2e-3)
    assert dp < (1e-4 if engine == "simt" else 1e-3)


def node_run(engine, factor, what, bs, **kw):
    m = freeze(module(engine, style="node", factor=factor), what)
    tr = D.FusedTrainer(m, lr=1e-3, weight_decay=1e-2, **kw)
    losses, rows = [], []
    for b in bs:
        losses.append(float(tr.step(b.to(DEV))))
        rows.append(tr.last_loss_rows().cpu())
    return losses, m, rows, tr


def node_reference(engine, factor, what, bs, rows_per_step):
    m = freeze(module(engine, style="node", factor=factor), what)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-2)
    losses = []
    for b, rows in zip(bs, rows_per_step):
        opt.zero_grad()
        b = b.to(DEV)
        out, label = m(b), m.get_label(b)
        idx = rows.long().to(DEV)
        loss = m.loss_fn(out[idx], label[idx])
        loss.backward()
        opt.step()
        losses.append(float(loss))
    return losses, m


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("factor", [None, 1.0])
@pytest.mark.parametrize("what", ["encoder", "tables"])
def test_node_style_follows_torch_adam(engine, factor, what):
    bs = [synth.make_batch(12, 40, seed=300 + i, variable=True, vuln_rate=0.5) for i in range(20)]
    lf, mf, rows, tr = node_run(engine, factor, what, bs)
    assert tr._grad_ggnn == (what != "encoder")
    lr_, mr = node_reference(engine, factor, what, bs, rows)
    assert_frozen_unchanged(mf, 1, engine, what, style="node", factor=factor)
    dl = max(abs(a - b) / max(1.0, abs(b)) for a, b in zip(lf, lr_))
    dp = max(float((p - q).abs().max()) for p, q in zip(mf.parameters(), mr.parameters()))
    print(f"node {engine} factor={factor} frozen={what}: max rel |dloss| {dl:.2e}, max |dparam| {dp:.2e}")
    assert dl < (2e-5 if engine == "simt" else 2e-3)
    assert dp < (2e-4 if engine == "simt" else 1e-3)


# ---- 4. step paths and modes --------------------------------------------------------------------------------------------
def params_and_state(m, tr):
    torch.cuda.synchronize()
    return [p.detach().clone() for p in m.parameters()], tr.exp_avg.clone(), tr.exp_avg_sq.clone(), int(tr.step_count)


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_captured_and_arena_steps_equal_the_eager_step(engine):
    with det_mode():
        dev_bs = [b.to(DEV) for b in [synth.make_batch(16, 40, seed=40 + i % 2, vuln_rate=0.3) for i in range(6)]]
        le, me, te = fused_graph(engine, "encoder", dev_bs)
        lc, mc, tc = fused_graph(engine, "encoder", dev_bs, use_cuda_graph=True)
        assert len(tc._graphs) >= 1
        assert le == lc
        for a, b in zip(params_and_state(me, te)[0], params_and_state(mc, tc)[0]):
            assert torch.equal(a, b)
        graphs = [synth.make_batch(1, 30, seed=600 + i, vuln_rate=0.3) for i in range(30)]
        arena = D.GraphArena.from_graphs(graphs, DEV)
        ids = [np.random.default_rng(i % 2).integers(0, 30, 8) for i in range(5)]
        m1, m2 = freeze(module(engine), "encoder"), freeze(module(engine), "encoder")
        t1, t2 = D.FusedTrainer(m1, use_cuda_graph=True), D.FusedTrainer(m2)
        for i in ids:
            assert float(t1.step_ids(arena, i)) == float(t2.step(arena.batch(i)))
        assert all(torch.equal(p, q) for p, q in zip(m1.parameters(), m2.parameters()))


def test_bucketed_host_stream_follows_the_eager_step():
    bs = graph_batches(8, seed=400, graphs=12, nodes=30)
    lb, mb, tb = fused_graph("tcgen05", "encoder", bs + bs, use_cuda_graph=True, bucket_nodes=64, bucket_edges=256,
                             bucket_min_pad_nodes=8, max_graph_shapes=16)
    assert tb.num_bucket_shapes() >= 2
    le2, me2, _ = fused_graph("tcgen05", "encoder", bs + bs)
    for a, b in zip(le2, lb):
        assert abs(a - b) < 2e-5 * max(1.0, abs(a))
    for p, q in zip(me2.parameters(), mb.parameters()):
        assert float((p - q).abs().max()) < 5e-4


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_clipping_norm_is_clip_grad_norm_of_the_model(engine):
    bs = graph_batches(3, seed=720)
    probe = freeze(module(engine, seed=2), "encoder")
    probe.training_step((bs[0].to(DEV), {}), 0).backward()
    bound = 0.25 * float(torch.nn.utils.clip_grad_norm_(probe.parameters(), float("inf")))
    _, mr, _, norms = reference_graph(engine, "encoder", bs, max_norm=bound)
    m = freeze(module(engine, seed=2), "encoder")
    tr = D.FusedTrainer(m, max_grad_norm=bound)
    for i, b in enumerate(bs):
        tr.step(b.to(DEV))
        torch.cuda.synchronize()
        assert abs(float(tr.grad_norm) - norms[i]) <= 1e-4 * norms[i], (i, float(tr.grad_norm), norms[i])
    assert norms[0] > bound
    assert max(float((p - q).abs().max()) for p, q in zip(m.parameters(), mr.parameters())) < 1e-3


def test_nan_step_is_skipped_bit_exactly():
    bs = [b.to(DEV) for b in graph_batches(2, seed=41)]
    m = freeze(module(seed=9), "encoder")
    tr = D.FusedTrainer(m, skip_nonfinite=True, max_grad_norm=5.0)
    tr.step(bs[0])
    before = params_and_state(m, tr)
    table = m.param_list()[0]
    keep = table.data.clone()
    with torch.no_grad():
        table.data.fill_(float("nan"))               # a frozen table: every logit and so every head gradient is NaN
    tr.step(bs[1])
    torch.cuda.synchronize()
    with torch.no_grad():
        table.data.copy_(keep)
    after = params_and_state(m, tr)
    assert tr.skipped_steps == 1
    assert all(torch.equal(a, b) for a, b in zip(before[0], after[0]))
    assert torch.equal(before[1], after[1]) and torch.equal(before[2], after[2]) and before[3] == after[3]


@pytest.mark.parametrize("style", ["graph", "node"])
def test_deterministic_frozen_runs_are_bit_identical(style):
    bs = [b.to(DEV) for b in graph_batches(6, seed=77)]
    runs = []
    with det_mode():
        for _ in range(2):
            m = freeze(module(style=style, factor=1.0 if style == "node" else None), "encoder")
            tr = D.FusedTrainer(m, node_sample_seed=3)
            losses = [float(tr.step(b)) for b in bs]
            runs.append((losses, params_and_state(m, tr)))
    (la, sa), (lb, sb) = runs
    assert all(a == b or (a != a and b != b) for a, b in zip(la, lb))
    assert all(torch.equal(a, b) for a, b in zip(sa[0], sb[0]))
    assert torch.equal(sa[1], sb[1]) and torch.equal(sa[2], sb[2]) and sa[3] == sb[3]


# ---- 5. state ------------------------------------------------------------------------------------------------------------
def test_state_dict_matches_torch_and_a_torch_checkpoint_resumes():
    bs = graph_batches(10, seed=800)
    _, mr, opt, _ = reference_graph("simt", "encoder", bs[:5])
    _, mf, tr = fused_graph("simt", "encoder", bs[:5])
    sd_t, sd_f = opt.state_dict(), tr.optimizer.state_dict()
    assert sorted(sd_f["state"]) == sorted(sd_t["state"])
    frozen = {i for i, p in enumerate(mf.parameters()) if not p.requires_grad}
    assert frozen and not frozen & set(sd_f["state"])
    for i, st in sd_t["state"].items():
        assert float(sd_f["state"][i]["step"]) == float(st["step"]) == 5.0
        for k in ("exp_avg", "exp_avg_sq"):
            assert sd_f["state"][i][k].shape == st[k].shape
    # resume the torch run in a fused trainer and continue it along the torch run
    m2 = freeze(module("simt", seed=99), "encoder")
    m2.load_state_dict(copy.deepcopy(mr.state_dict()))
    tr2 = D.FusedTrainer(m2, lr=1e-3, weight_decay=1e-2)
    tr2.optimizer.load_state_dict(copy.deepcopy(sd_t))
    assert int(tr2.step_count) == 5
    for b in bs[5:]:
        opt.zero_grad()
        mr.training_step((b.to(DEV), {}), 0).backward()
        opt.step()
        tr2.step(b.to(DEV))
    assert max(float((p - q).abs().max()) for p, q in zip(m2.parameters(), mr.parameters())) < 1e-4


# ---- 6. errors -----------------------------------------------------------------------------------------------------------
def test_changing_requires_grad_after_construction_raises():
    b = graph_batches(1)[0].to(DEV)
    m = freeze(module(), "encoder")
    tr = D.FusedTrainer(m, use_cuda_graph=True)
    tr.step(b)
    m.ggnn.gru.weight_hh.requires_grad_(True)
    with pytest.raises(ValueError, match="build a new FusedTrainer"):
        tr.step(b)
    m.ggnn.gru.weight_hh.requires_grad_(False)
    tr.step(b)
    m2 = module()
    for p in m2.parameters():
        p.requires_grad_(False)
    with pytest.raises(ValueError, match="nothing to train"):
        D.FusedTrainer(m2)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, q):
    import torch.distributed as dist
    from deepdfa_b200.batched_graph import split_batch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    try:
        full = [synth.make_batch(48, 60, seed=900 + i, variable=True, vuln_rate=0.3) for i in range(5)]
        m_dp = freeze(module("tcgen05", seed=4, device=dev), "encoder")
        tr_dp = D.FusedTrainer(m_dp, distributed=True, exchange="auto")
        m_1 = freeze(module("tcgen05", seed=4, device=dev), "encoder")
        tr_1 = D.FusedTrainer(m_1, distributed=False)
        l_dp, l_1 = [], []
        for b in full:
            l_dp.append(float(tr_dp.step(split_batch(b, 2)[rank].to(dev), global_batch=b.batch_size)))
            l_1.append(float(tr_1.step(b.to(dev), global_batch=b.batch_size)))
        dp = max(float((p - r).abs().max()) for p, r in zip(m_dp.parameters(), m_1.parameters()))
        q.put((rank, (tr_dp.exchange, tr_dp.exchange_note, l_dp, l_1, dp)))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


def test_two_ranks_nccl_with_a_frozen_encoder_match_one_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, q)) for r in range(2)]
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
    for r in (0, 1):
        assert not isinstance(res[r], str), res[r]
        exchange, note, l_dp, l_1, dp = res[r]
        assert exchange == "nccl" and "frozen" in note
        assert max(abs(a - b) for a, b in zip(l_dp, l_1)) < 1e-4
        assert dp < 1e-4


# ---- 7. memory -----------------------------------------------------------------------------------------------------------
def step_peak_bytes(what, b):
    """Peak allocated memory a C1 step adds on top of what was allocated before it (module, trainer buffers, batch)."""
    m = module("tcgen05", seed=0, steps=8, graphs_hidden=32)
    if what != "none":
        freeze(m, what)
    tr = D.FusedTrainer(m)
    g = b.to(DEV)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    tr.step(g, global_batch=b.batch_size)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del tr, m, g
    gc.collect()
    torch.cuda.empty_cache()
    return peak


def test_frozen_encoder_step_needs_a_quarter_of_the_memory_at_c1():
    b = synth.make_batch(1024, 150, seed=1)
    full = step_peak_bytes("none", b)
    frozen = step_peak_bytes("encoder", b)
    print(f"C1 step peak: all trainable {full / 2**20:.0f} MiB, encoder frozen {frozen / 2**20:.0f} MiB ({frozen / full:.1%})")
    assert frozen <= 0.25 * full
