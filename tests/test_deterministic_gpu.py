"""GPU: deterministic mode (DDFA_TUNE_DETERMINISTIC = 1) gives bit-identical results from identical inputs and state.

Checked: the deterministic embedding backward at a hub batch (index 0 on ~75 % of the nodes) against fp64 and against itself; the
readout / MLP / loss reductions at B = 1, B < 256 and B >= 256; whole FusedTrainer runs at the benchmark's C1 size (eager,
captured, arena; host batch against arena; resume from a checkpoint); the module path under torch.use_deterministic_algorithms;
and a trainer whose graphs were captured in the default mode before the mode was switched on."""
import contextlib
import os
import socket

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200 import engine as E
from deepdfa_b200._lib import lib, ptr_array

from scale_batches import hub_batch

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


@contextlib.contextmanager
def tuning(key, value):
    prev = lib().call("ddfa_tuning_get", key)
    lib().call("ddfa_tuning_set", key, value)
    try:
        yield
    finally:
        lib().call("ddfa_tuning_set", key, prev)


def new_module(engine="tcgen05", seed=1):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine).to(DEV)


def grads_of(m, batch):
    m.zero_grad(set_to_none=True)
    loss = m.training_step((batch, None))
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), [p.grad.detach().clone() for p in m.parameters()]


# ---- 1. the embedding backward: repeatable, and within fp64 bounds -----------------------------------------------------
@pytest.mark.parametrize("N", [100, 128 * 40 + 1, 157_381])
def test_embedding_backward_is_repeatable_and_accurate(N):
    g = torch.Generator().manual_seed(N)
    K, V, H = 4, 1002, 32
    idx = []
    for k in range(K):
        v = torch.randint(2, V, (N,), generator=g)
        r = torch.rand(N, generator=g)
        v[r < 0.75] = 0                      # index 0 on ~75 % of nodes, index 1 on a few %, as synth draws them
        v[(r >= 0.75) & (r < 0.78)] = 1
        idx.append(v.to(DEV))
    dx = torch.randn(N, K * H, generator=g).to(DEV)
    dx2 = torch.randn(N, K * H, generator=g).to(DEV)
    nbytes = lib().call("ddfa_embed_concat_bwd_workspace_bytes", K, V, H, N)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    outs = []
    with det_mode():
        _lib.apply_deterministic_mode()
        for _ in range(2):
            dt = [torch.full((V, H), 0.5, device=DEV) for _ in range(K)]
            ws.fill_(0xAB)                   # stale scratch must not matter
            lib().call("ddfa_embed_concat_bwd_ws", ptr_array([t.data_ptr() for t in idx]), dx.data_ptr(), dx2.data_ptr(), K, V, H, N,
                       ptr_array([t.data_ptr() for t in dt]), ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream)
            outs.append(dt)
        torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    s = (dx + dx2).double()
    for k in range(K):
        ref = torch.full((V, H), 0.5, dtype=torch.float64, device=DEV).index_add_(0, idx[k], s[:, k * H:(k + 1) * H])
        scale = torch.zeros(V, H, dtype=torch.float64, device=DEV).index_add_(0, idx[k], s[:, k * H:(k + 1) * H].abs())
        err = (outs[0][k].double() - ref).abs()
        assert bool((err <= 1e-5 * scale + 1e-6).all()), float((err / (scale + 1e-6)).max())


# ---- 2. whole backward passes of the module path: every gradient bit-identical, close to the default mode -----------------
@pytest.mark.parametrize("engine,gate_bwd_tma", [("tcgen05", 0), ("tcgen05", 1), ("tcgen05", 2), ("simt", 2)])
@pytest.mark.parametrize("B", [1, 100, 300])
def test_module_backward_is_repeatable(B, engine, gate_bwd_tma, monkeypatch):
    batch = synth.make_batch(B, 150, seed=B, variable=True, vuln_rate=0.3).to(DEV)
    m = new_module(engine)
    prev = torch.are_deterministic_algorithms_enabled()
    monkeypatch.delenv("DDFA_DETERMINISTIC", raising=False)
    with tuning(_lib.TUNE_GATE_BWD_TMA, gate_bwd_tma):
        try:
            torch.use_deterministic_algorithms(True)
            l1, g1 = grads_of(m, batch)
            l2, g2 = grads_of(m, batch)
        finally:
            torch.use_deterministic_algorithms(prev)
            _lib.apply_deterministic_mode()
        l0, g0 = grads_of(m, batch)          # default mode
    assert l1 == l2 and all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert abs(l1 - l0) <= 1e-5 * max(1.0, abs(l0))
    for a, b in zip(g1, g0):
        assert float((a - b).abs().max()) <= 1e-4 * max(1.0, float(b.abs().max()))


def test_fp32_saved_state_backward_is_repeatable():
    batch = synth.make_batch(64, 150, seed=5, variable=True, vuln_rate=0.3).to(DEV)
    m = new_module()
    prev = E.OPTIONS["packed_state"]
    try:
        E.OPTIONS["packed_state"] = False
        with det_mode():
            r1, r2 = grads_of(m, batch), grads_of(m, batch)
    finally:
        E.OPTIONS["packed_state"] = prev
    assert r1[0] == r2[0] and all(torch.equal(a, b) for a, b in zip(r1[1], r2[1]))


def test_hub_batch_backward_is_repeatable():
    batch = hub_batch("threshold").to(DEV)
    m = new_module()
    with det_mode():
        r1, r2 = grads_of(m, batch), grads_of(m, batch)
    assert r1[0] == r2[0] and all(torch.equal(a, b) for a, b in zip(r1[1], r2[1]))


# ---- 3. whole FusedTrainer runs at C1 --------------------------------------------------------------------------------------
C1 = dict(num_graphs=1024, nodes_per_graph=150, variable=True, vuln_rate=0.3)


def c1_batches(n=3):
    return [synth.make_batch(seed=100 + i, **C1) for i in range(n)]


def state_of(tr, losses):
    torch.cuda.synchronize()
    return losses, [t.detach().clone() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]


def assert_same(a, b):
    assert a[0] == b[0], (a[0], b[0])
    for x, y in zip(a[1], b[1]):
        assert torch.equal(x, y)


def run(mode, steps=20, batches=None, arena_ids=None, ckpt_at=None, tmp_path=None, engine="tcgen05"):
    m = new_module(engine, seed=7)
    tr = D.FusedTrainer(m, use_cuda_graph=mode != "eager")
    losses = []
    for i in range(steps):
        if ckpt_at is not None and i == ckpt_at:
            torch.save({"state_dict": m.state_dict(), "optimizer": tr.optimizer.state_dict()}, tmp_path / "ckpt.pt")
            ck = torch.load(tmp_path / "ckpt.pt", weights_only=True)
            m = new_module(engine, seed=99)
            tr = D.FusedTrainer(m, use_cuda_graph=mode != "eager")
            m.load_state_dict(ck["state_dict"])
            tr.optimizer.load_state_dict(ck["optimizer"])
        if mode == "arena":
            losses.append(float(tr.step_ids(batches, arena_ids[i % len(arena_ids)])))
        else:
            b = batches[i % len(batches)]
            losses.append(float(tr.step(b.to(DEV) if mode == "eager" and not isinstance(b, D.ArenaBatch) else b)))
    return state_of(tr, losses)


@pytest.mark.parametrize("mode", ["eager", "graph", "resident"])
def test_trainer_runs_are_bit_identical(mode):
    bs = c1_batches()
    if mode == "resident":
        bs = [b.to(DEV) for b in bs]
    with det_mode():
        a = run("graph" if mode == "resident" else mode, batches=bs)
        b = run("graph" if mode == "resident" else mode, batches=bs)
    assert_same(a, b)


def test_eager_and_captured_steps_are_bit_identical():
    bs = c1_batches()
    with det_mode():
        assert_same(run("eager", steps=6, batches=bs), run("graph", steps=6, batches=bs))


def test_arena_runs_and_host_batches_over_the_same_ids_are_bit_identical():
    graphs = [synth.make_batch(1, 150, seed=3000 + i, vuln_rate=0.5) for i in range(2048)]
    rng = np.random.default_rng(0)
    ids = [rng.choice(2048, 1024, replace=False) for _ in range(3)]
    arena = D.GraphArena.from_graphs(graphs, DEV)
    with det_mode():
        a = run("arena", batches=arena, arena_ids=ids)
        b = run("arena", batches=arena, arena_ids=ids)
        assert_same(a, b)
        host = [D.batch([graphs[j] for j in i]) for i in ids]     # the same graphs collated on the host: CSR from ddfa_build_csr
        c = run("graph", steps=6, batches=host)
        d = run("arena", steps=6, batches=arena, arena_ids=ids)
    assert_same(c, d)


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_resume_is_bit_identical_to_the_uninterrupted_run(mode, tmp_path):
    bs = c1_batches()
    with det_mode():
        a = run(mode, batches=bs)
        b = run(mode, batches=bs, ckpt_at=10, tmp_path=tmp_path)
    assert_same(a, b)


def test_switching_the_mode_on_replays_no_graph_of_the_default_mode():
    bs = c1_batches()
    m = new_module(seed=7)
    tr = D.FusedTrainer(m, use_cuda_graph=True)
    with det_mode(False):
        for i in range(4):                       # warm-up + capture in the default mode
            tr.step(bs[i % 3])
    torch.cuda.synchronize()
    start = {k: v.detach().clone() for k, v in m.state_dict().items()}
    opt = tr.optimizer.state_dict()
    with det_mode():
        got = state_of(tr, [float(tr.step(bs[i % 3])) for i in range(4)])
        m2 = new_module(seed=99)
        tr2 = D.FusedTrainer(m2, use_cuda_graph=True)
        m2.load_state_dict(start)
        tr2.optimizer.load_state_dict(opt)
        want = state_of(tr2, [float(tr2.step(bs[i % 3])) for i in range(4)])
    assert_same(got, want)


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_simt_engine_trainer_runs_are_bit_identical(mode, tmp_path):
    bs = [synth.make_batch(256, 150, seed=200 + i, variable=True, vuln_rate=0.3) for i in range(3)]
    with det_mode():
        a = run(mode, steps=8, batches=bs, engine="simt")
        b = run(mode, steps=8, batches=bs, engine="simt", ckpt_at=4, tmp_path=tmp_path)
    assert_same(a, b)


# ---- 4. entry points without a deterministic form --------------------------------------------------------------------------
def test_old_entry_points_refuse_deterministic_mode():
    with det_mode():
        _lib.apply_deterministic_mode()
        with pytest.raises(_lib.DdfaError, match="ddfa_embed_concat_bwd_ws"):
            lib().call("ddfa_embed_concat_bwd", None, None, None, 4, 1002, 32, 1, None, None)
        with pytest.raises(_lib.DdfaError, match="ddfa_readout_bwd_ws"):
            lib().call("ddfa_readout_bwd", *([None] * 5), 1, 128, *([None] * 8), None)


# ---- 5. two GPUs, exchange="p2p" -------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _p2p_worker(rank, port, q):
    """Two uninterrupted deterministic runs per rank; both ranks make the same collective calls and assert nothing here."""
    import torch.distributed as dist
    from deepdfa_b200.batched_graph import split_batch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2", DDFA_DETERMINISTIC="1")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    out = {}
    try:
        full = [synth.make_batch(256, 150, seed=900 + i, variable=True, vuln_rate=0.3) for i in range(3)]
        shards = [split_batch(b, 2)[rank].to(dev) for b in full]
        for name in ("A", "B"):
            torch.manual_seed(7)
            m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, positive_weight=2.0, engine="tcgen05").to(dev)
            tr = D.FusedTrainer(m, distributed=True, exchange="p2p")
            losses = [float(tr.step(shards[i % 3], global_batch=256)) for i in range(10)]
            torch.cuda.synchronize()
            out[name] = (losses, [t.detach().cpu() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)])
        q.put((rank, out))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


def test_two_ranks_p2p_runs_are_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_p2p_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = {}
    try:
        for _ in range(2):
            rank, out = q.get(timeout=600)
            results[rank] = out
    finally:
        for p in procs:
            p.join(timeout=120)
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(timeout=30)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for rank in (0, 1):
        assert not isinstance(results[rank], str), results[rank]
        assert_same(results[rank]["A"], results[rank]["B"])
