"""GPU: gradient accumulation in FusedTrainer (accumulate_grad_batches=k): micro-batch gradients summed on the device, one
exchange, guard and Adam update per window.

Checked: k = 1 enqueues what a trainer without the argument enqueues and trains bit-identically; the window's arithmetic is exact
(two halves of one batch make one step; a window of two batches is Adam over their summed gradient); k = 4 follows the fp64
oracle doing (loss / 4).backward() four times per opt.step(); every step path gives the same bits; the guard acts on the window's
sum and skips a non-finite window whole; frozen tensors stay put; an LR schedule stepped per window reaches captured launches;
flush() applies a partial window; and with two GPUs the exchange runs once per window."""
import contextlib
import copy
import gc
import math
import os
import socket

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200._lib import lib
from deepdfa_b200.engine import _p, _stream_ptr
from oracle import ggnn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


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


def engines():
    return ["simt", "tcgen05"] if lib().call("ddfa_engine_available", 1) else ["simt"]


def module(style="graph", engine="simt", seed=1, factor=None, device=DEV):
    torch.manual_seed(seed)
    kw = dict(label_style="node", undersample_node_on_loss_factor=factor) if style == "node" else {}
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine, **kw).to(device)


def batches(n, seed=100, graphs=16, nodes=40, variable=True):
    return [synth.make_batch(graphs, nodes, seed=seed + i, variable=variable, vuln_rate=0.4) for i in range(n)]


def state(tr):
    torch.cuda.synchronize()
    return [t.detach().clone() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]


def assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (i, float((x.double() - y.double()).abs().max()))


def cuda_kernels(fn):
    """The names of the device activities ``fn`` enqueues (sorted) and the library's launch count over it.  Earlier work
    finishes and the garbage earlier tests left is collected first, so neither is recorded in the window."""
    from torch.profiler import ProfilerActivity, profile
    gc.collect()
    torch.cuda.synchronize()
    n0 = lib().call("ddfa_launch_count")
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = sorted(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return names, lib().call("ddfa_launch_count") - n0


def skip_missing(engine):
    if engine not in engines():
        pytest.skip("tcgen05 engine not compiled in")


# ---- 1. k = 1 is the trainer as it was -----------------------------------------------------------------------------------
@pytest.mark.parametrize("style", ["graph", "node"])
def test_k1_enqueues_what_the_trainer_without_the_argument_enqueues(style):
    b = batches(1)[0].to(DEV)
    seen = []
    for kw in ({}, {"accumulate_grad_batches": 1}):
        tr = D.FusedTrainer(module(style, factor=1.0), **kw)
        assert tr._acc is None and tr.accumulated == 0
        tr.step(b)                                            # warm-up: workspace growth
        tr.step(b)                                            # capture (its gc.collect / empty_cache stay out of the window)
        names, launches = cuda_kernels(lambda: tr.step(b))    # the step every later step replays
        assert tr.accumulated == 0
        seen.append((names, launches))
    assert seen[0][1] > 0 and seen[0] == seen[1]
    assert not any("accumulate" in n for n in seen[1][0])


@pytest.mark.parametrize("style", ["graph", "node"])
@pytest.mark.parametrize("captured", [False, True])
def test_k1_runs_are_bit_identical_to_runs_without_the_argument(style, captured):
    bs = batches(3, variable=False)
    out = []
    with det_mode():
        for kw in ({}, {"accumulate_grad_batches": 1}):
            tr = D.FusedTrainer(module(style, factor=1.0), use_cuda_graph=captured, node_sample_seed=2, **kw)
            losses = [float(tr.step(bs[i % 3] if captured else bs[i % 3].to(DEV))) for i in range(8)]
            out.append((losses, state(tr), sorted(tr._stream_slots)))
    assert out[0][0] == out[1][0]
    assert_same(out[0][1], out[1][1])
    assert out[0][2] == out[1][2]
    if captured:
        assert all(st["graph"] is not None for slot in tr._stream_slots.values() for st in slot["sets"])


# ---- 2. the window's arithmetic is exact -------------------------------------------------------------------------------------
def assert_no_subnormal(g):
    tiny = torch.finfo(torch.float32).tiny
    bad = int(((g != 0) & (g.abs() < 2 * tiny)).sum())
    assert bad == 0, f"premise: the k = 1 gradient has {bad} entries whose half is an fp32 subnormal; halving them is not exact"


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("style", ["graph", "node"])
def test_two_halves_of_one_batch_make_one_step(engine, style):
    skip_missing(engine)
    b = batches(1, graphs=24)[0].to(DEV)
    with det_mode():
        t1 = D.FusedTrainer(module(style, engine))
        l1 = float(t1.step(b))
        torch.cuda.synchronize()
        assert_no_subnormal(t1.flat_g[:t1.numel])
        t2 = D.FusedTrainer(module(style, engine), accumulate_grad_batches=2)
        la = float(t2.step(b))
        torch.cuda.synchronize()
        assert t2.accumulated == 1 and int(t2.step_count) == 0
        lb = float(t2.step(b))
        assert t2.accumulated == 0
    assert la == lb == l1                                 # the returned loss is the micro-batch's own mean, undivided
    assert_same(state(t1), state(t2))


def flat_grads(engine, bs, global_batch):
    """The initial flat parameters and flat_g after each step of a k = 1 trainer that does not move (lr = 0, no decay)."""
    tr = D.FusedTrainer(module("graph", engine), lr=0.0, weight_decay=0.0)
    p0 = tr.flat_p.detach().clone()
    gs = []
    for b in bs:
        tr.step(b.to(DEV), global_batch=global_batch)
        torch.cuda.synchronize()
        gs.append(tr.flat_g[:tr.numel].detach().clone())
    assert torch.equal(tr.flat_p, p0), "premise: lr = 0 leaves the parameters where they were"
    return p0, gs


def adam_from_start(tr, p0, g):
    """One ddfa_adam_flat_hp step from p0 and zero moments on the gradient g, with tr's hyperparameters."""
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    lib().call("ddfa_adam_flat_hp", _p(p), _p(g), _p(m), _p(v), _p(step), p.numel(), _p(tr.hyper), _stream_ptr())
    torch.cuda.synchronize()
    return [p, m, v, step]


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_a_window_of_two_batches_is_adam_over_their_summed_gradients(engine):
    skip_missing(engine)
    A, B = batches(2, seed=300)
    with det_mode():
        p0, (gA, gB) = flat_grads(engine, [A, B], 2 * 16)
        tr = D.FusedTrainer(module("graph", engine), accumulate_grad_batches=2)
        tr.step(A.to(DEV), global_batch=16)
        tr.step(B.to(DEV), global_batch=16)
        want = adam_from_start(tr, p0, gA + gB)
    assert_same(state(tr), want)


# ---- 3. against the fp64 oracle ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine,style", [("simt", "graph"), ("tcgen05", "graph"), ("simt", "node")])
def test_k4_tracks_the_oracle_accumulating_loss_over_4(engine, style):
    skip_missing(engine)
    torch.manual_seed(0)
    o = O.OracleFlowGNNGGNN(FEAT, 1002, 32, 5, 3, concat_all_absdf=True, positive_weight=8.0, label_style=style)
    kw = dict(label_style="node", undersample_node_on_loss_factor=None) if style == "node" else {}
    m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 5, 3, concat_all_absdf=True, positive_weight=8.0, engine=engine, **kw)
    m.load_state_dict(copy.deepcopy(o.state_dict()))
    m.to(DEV)
    o = o.double()
    tr = D.FusedTrainer(m, accumulate_grad_batches=4)
    opt = O.make_optimizer(o)
    bs = [synth.make_batch(32, 60, seed=50 + i, variable=True, vuln_rate=0.3) for i in range(12)]     # 3 windows
    for i, b in enumerate(bs):
        if i % 4 == 0:
            opt.zero_grad()
        loss_ref, _ = o.training_loss(b)
        (loss_ref / 4).backward()
        if i % 4 == 3:
            opt.step()
        loss = float(tr.step(b))
        assert abs(loss - float(loss_ref)) < 2e-3 * max(1.0, abs(float(loss_ref))), (i, loss, float(loss_ref))
    assert int(tr.step_count) == 3
    with torch.no_grad():
        ref = o(bs[0]).double()
        out = m(bs[0], {})
    assert (out.cpu().double() - ref).abs().max() < 5e-3


# ---- 4. every step path gives the same bits ------------------------------------------------------------------------------------
def test_step_paths_agree_bit_for_bit_over_windows():
    graphs = [synth.make_batch(1, 40, seed=3000 + i, variable=True, vuln_rate=0.4) for i in range(64)]
    arena = D.GraphArena.from_graphs(graphs, DEV)
    rng = np.random.default_rng(0)
    ids = [rng.choice(64, 16, replace=False) for _ in range(2)]
    host = [D.batch([graphs[j] for j in i]) for i in ids]
    assert (host[0].num_nodes(), host[0].num_edges()) != (host[1].num_nodes(), host[1].num_edges())
    resident = [b.to(DEV) for b in host]
    pinned = [b.pin_memory() for b in host]
    steps = 18            # 6 windows of k = 3 over 2 batches: every (shape, phase) pair is visited three times
    runs = {}
    with det_mode():
        for mode in ("eager", "host", "prefetch", "resident", "arena"):
            tr = D.FusedTrainer(module(seed=4), use_cuda_graph=mode != "eager", accumulate_grad_batches=3)
            losses = []
            for i in range(steps):
                if mode == "eager":
                    loss = tr.step(resident[i % 2])
                elif mode == "host":
                    loss = tr.step(host[i % 2])
                elif mode == "prefetch":
                    loss = tr.step(pinned[i % 2])
                    tr.prefetch(pinned[(i + 1) % 2])
                elif mode == "resident":
                    loss = tr.step(resident[i % 2])
                else:
                    loss = tr.step_ids(arena, ids[i % 2])
                losses.append(float(loss))
            runs[mode] = (losses, state(tr))
            if mode in ("host", "prefetch"):
                assert len(tr._stream_slots) == 6            # 2 shapes x 3 phases, each with both buffer sets captured
                assert all(st["graph"] is not None for slot in tr._stream_slots.values() for st in slot["sets"])
            if mode == "resident":
                assert len(tr._graphs) == 6
            if mode == "arena":
                assert len(tr._stream_slots) == 6 and all(s["graph"] is not None for s in tr._stream_slots.values())
    for mode in ("host", "prefetch", "resident", "arena"):
        assert runs[mode][0] == runs["eager"][0], mode
        assert_same(runs[mode][1], runs["eager"][1])
    assert int(runs["eager"][1][3]) == steps // 3


def test_bucketed_host_stream_follows_the_eager_windows():
    """Bucketing pads every batch with a dummy graph (other tile shapes, other fp32 sums): close to eager, not bit-equal."""
    bs = batches(4, seed=500)
    out = {}
    for mode in ("eager", "bucketed"):
        kw = dict(use_cuda_graph=True, bucket_nodes=256, bucket_edges=1024, bucket_min_pad_nodes=8) if mode == "bucketed" else {}
        tr = D.FusedTrainer(module(seed=6), accumulate_grad_batches=3, **kw)
        losses = [float(tr.step(bs[i % 4] if mode == "bucketed" else bs[i % 4].to(DEV))) for i in range(12)]
        out[mode] = (losses, state(tr), tr)
    tr = out["bucketed"][2]
    assert tr.num_bucket_shapes() >= 1 and any(st["graph"] is not None for s in tr._stream_slots.values() for st in s["sets"])
    for a, b in zip(out["eager"][0], out["bucketed"][0]):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(a))
    assert float((out["eager"][1][0] - out["bucketed"][1][0]).abs().max()) <= 1e-5
    assert int(out["bucketed"][1][3]) == 4


# ---- 5. guard and frozen parameters -------------------------------------------------------------------------------------------
def test_max_grad_norm_clips_the_window_sum():
    A, B = batches(2, seed=700)
    with det_mode():
        p0, (gA, gB) = flat_grads("simt", [A, B], 2 * 16)
        tr = D.FusedTrainer(module(), accumulate_grad_batches=2, max_grad_norm=0.01)
        tr.step(A.to(DEV), global_batch=16)
        tr.step(B.to(DEV), global_batch=16)
        torch.cuda.synchronize()
    ref = math.sqrt(float(((gA + gB).double() ** 2).sum()))
    assert ref > 0.01, "the bound must bite"
    assert abs(float(tr.grad_norm) - ref) <= 1e-5 * ref
    assert int(tr.step_count) == 1


def test_a_nonfinite_window_is_skipped_whole_and_the_run_continues_as_if_it_never_happened():
    bs = [b.to(DEV) for b in batches(6, seed=800, variable=False)]
    runs = {}
    with det_mode():
        for poisoned in (False, True):
            m = module(seed=9)
            tr = D.FusedTrainer(m, accumulate_grad_batches=2, skip_nonfinite=True, max_grad_norm=5.0)
            tr.step(bs[0])
            tr.step(bs[1])
            if poisoned:
                table = m.param_list()[0]                 # embedding table 0: row 0 is the index of most nodes
                keep = table.data[0].clone()
                with torch.no_grad():
                    table.data[0] = float("nan")
                tr.step(bs[2])                            # the window's first micro-batch sees the NaN
                torch.cuda.synchronize()
                with torch.no_grad():
                    table.data[0] = keep
                tr.step(bs[3])                            # the second is clean: the window's sum is still NaN
                torch.cuda.synchronize()
                assert not math.isfinite(float(tr.grad_norm))
            tr.step(bs[4])
            tr.step(bs[5])
            runs[poisoned] = (state(tr), tr.skipped_steps)
    (a, skipped_a), (b, skipped_b) = runs[False], runs[True]
    assert skipped_a == 0 and skipped_b == 1
    assert_same(a, b)
    assert int(b[3]) == 2


def test_frozen_tensors_stay_put_across_windows():
    m = module(seed=3)
    frozen = [m.param_list()[0], m.param_list()[-1]]
    for p in frozen:
        p.requires_grad_(False)
    before = [p.detach().clone() for p in frozen]
    moving = m.param_list()[-3]
    start = moving.detach().clone()
    tr = D.FusedTrainer(m, accumulate_grad_batches=3, max_grad_norm=1.0)
    bs = [b.to(DEV) for b in batches(3, seed=900)]
    for i in range(6):
        tr.step(bs[i % 3])
    torch.cuda.synchronize()
    assert all(torch.equal(p.detach(), q) for p, q in zip(frozen, before))
    assert not torch.equal(moving.detach(), start)
    assert int(tr.step_count) == 2


# ---- 6. schedules and flush -------------------------------------------------------------------------------------------------
def test_an_lr_schedule_stepped_per_window_reaches_captured_launches():
    bs = batches(3, seed=1000, variable=False)
    out = {}
    with det_mode():
        for captured in (False, True):
            tr = D.FusedTrainer(module(seed=5), use_cuda_graph=captured, accumulate_grad_batches=2)
            sched = torch.optim.lr_scheduler.LambdaLR(tr.optimizer, lambda s: 1.0 / (1 + s))
            for i in range(12):
                tr.step(bs[i % 3] if captured else bs[i % 3].to(DEV))
                if tr.accumulated == 0:
                    sched.step()
            out[captured] = (state(tr), tr.lr)
            if captured:
                assert all(st["graph"] is not None for s in tr._stream_slots.values() for st in s["sets"])
    assert_same(out[False][0], out[True][0])
    assert out[True][1] == out[False][1] == pytest.approx(1e-3 / 7)


def test_flush_applies_a_partial_window_and_nothing_on_an_empty_one():
    A, B = batches(2, seed=1100)
    with det_mode():
        p0, (gA, gB) = flat_grads("simt", [A, B], 4 * 16)
        tr = D.FusedTrainer(module(), accumulate_grad_batches=4)
        tr.step(A.to(DEV), global_batch=16)
        tr.step(B.to(DEV), global_batch=16)
        assert tr.accumulated == 2 and int(tr.step_count) == 0
        tr.flush()
        assert tr.accumulated == 0
        want = adam_from_start(tr, p0, gA + gB)
        assert_same(state(tr), want)
        names, launches = cuda_kernels(tr.flush)
    assert names == [] and launches == 0
    assert_same(state(tr), want)


# ---- 7. two GPUs: one exchange per window -------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, exchange, overlap, q):
    import torch.distributed as dist
    from deepdfa_b200.batched_graph import split_batch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2", DDFA_DETERMINISTIC="1")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    real = dist.all_reduce
    try:
        full = [synth.make_batch(64, 60, seed=900 + i, variable=True, vuln_rate=0.3) for i in range(4)]
        shards = [split_batch(b, 2)[rank].to(dev) for b in full]
        m = module(seed=7, device=dev)
        tr = D.FusedTrainer(m, distributed=True, exchange=exchange, overlap_allreduce=overlap, accumulate_grad_batches=2)
        calls = []

        def counting(*a, **k):
            calls.append(1)
            return real(*a, **k)
        dist.all_reduce = counting                      # the trainer's collectives go through torch.distributed.all_reduce
        per_step, losses = [], []
        for i in range(8):
            n = len(calls)
            losses.append(float(tr.step(shards[i % 4], global_batch=64)))
            per_step.append(len(calls) - n)
        torch.cuda.synchronize()
        dist.all_reduce = real
        m1 = module(seed=7, device=dev)
        t1 = D.FusedTrainer(m1, distributed=False, accumulate_grad_batches=2)
        l1 = [float(t1.step(full[i % 4].to(dev), global_batch=64)) for i in range(8)]
        torch.cuda.synchronize()
        dp = max(float((p.data - r.data).abs().max()) for p, r in zip(m.param_list(), m1.param_list()))
        q.put((rank, (per_step, losses, l1, dp, int(tr.step_count), tr.exchange)))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.all_reduce = real
        dist.destroy_process_group()


@pytest.mark.parametrize("exchange,overlap", [("nccl", True), ("nccl", False), ("p2p", True)])
def test_two_ranks_exchange_once_per_window_and_match_the_unsharded_windows(exchange, overlap):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, exchange, overlap, q)) for r in range(2)]
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
    for r in (0, 1):
        assert not isinstance(res[r], str), res[r]
    per_call = {("nccl", True): 3, ("nccl", False): 1, ("p2p", True): 0}[(exchange, overlap)]   # split: 2 small ranges + GEMM range
    for r in (0, 1):
        per_step, losses, l1, dp, steps, used = res[r]
        assert used == exchange
        assert per_step == [0, per_call] * 4
        assert steps == 4
        assert dp <= 1e-3, dp
        for i in range(1, 8, 2):                        # the applying micro-batch returns the global loss
            assert abs(losses[i] - l1[i]) <= 1e-5 * max(1.0, abs(l1[i])), (i, losses[i], l1[i])
    for i in range(0, 8, 2):                            # the others return this rank's share of it
        total = res[0][1][i] + res[1][1][i]
        assert abs(total - res[0][2][i]) <= 1e-5 * max(1.0, abs(res[0][2][i])), (i, total, res[0][2][i])
