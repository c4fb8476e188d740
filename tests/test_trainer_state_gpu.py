"""GPU: FusedTrainer runs that stop and resume, hand over to and from torch.optim.Adam, and follow LR schedules under CUDA graphs.

``trainer.optimizer`` (FusedAdam) moves the Adam state between the trainer's flat buffers and torch's format, and hands the
hyperparameters to the Adam kernels through a device word they read when they run (``ddfa_adam_flat_hp`` /
``ddfa_allreduce_adam_p2p_hp``).

Bit-exact checks: the hyperparameter entry points against the by-value ones, and the state a load puts into the buffers.
Whole training runs are compared differently.  Several backward kernels sum with float atomics, so two uninterrupted runs of
the same code can differ in the last bits, and those differences grow through Adam.  Such comparisons are therefore bounded by
the spread between two uninterrupted runs made in the same test (``assert_runs_match``).  When the kernels happen to sum in
the same order, that spread is zero, and the runs must then be bit-identical."""
import copy
import os
import socket
import warnings

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import synth
from deepdfa_b200._lib import lib, ptr_array
from deepdfa_b200.engine import _p, _stream_ptr
from deepdfa_b200.trainer import flat_offsets, owned_range

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_optimizer_golden.pt")


def new_module(engine="simt", seed=1, device=DEV):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine).to(device)


def new_trainer(engine="simt", seed=1, device=DEV, **kw):
    m = new_module(engine, seed, device)
    return m, D.FusedTrainer(m, **kw)


def host_batches(n=4, seed=700):
    return [synth.make_batch(16, 40, seed=seed + i, vuln_rate=0.3) for i in range(n)]     # one shape: one captured graph


def params_of(m):
    return [p.detach().clone() for p in m.parameters()]


def assert_runs_match(got, ref, ref2, what=""):
    """got / ref / ref2 = (losses, parameters).  ``got`` must be as close to ``ref`` as two uninterrupted runs are to each
    other (x4), plus a floor far below what a lost moment or a restarted bias correction does to one Adam step (~1e-3)."""
    (lg, pg), (lr_, pr), (lr2, pr2) = got, ref, ref2
    noise_l = max(abs(a - b) for a, b in zip(lr_, lr2))
    noise_p = max(float((a - b).abs().max()) for a, b in zip(pr, pr2))
    dl = max(abs(a - b) for a, b in zip(lg, lr_))
    dp = max(float((a - b).abs().max()) for a, b in zip(pg, pr))
    exact = lg == lr_ and all(torch.equal(a, b) for a, b in zip(pg, pr))
    print(f"{what}: |dloss| {dl:.2e} |dparam| {dp:.2e} (two uninterrupted runs: {noise_l:.2e} / {noise_p:.2e}), bit-identical: {exact}")
    assert dl <= 4 * noise_l + 1e-6, (what, lg, lr_)
    assert dp <= 4 * noise_p + 1e-5, (what, dp, noise_p)


class Workload:
    """The three ways to feed a FusedTrainer: eager device batches, host batches through captured per-shape graphs, and id
    lists over a device arena (``step_ids``; the host may run ahead)."""

    def __init__(self, mode):
        self.mode = mode
        self.host = host_batches()
        if mode == "arena":
            self.graphs = [synth.make_batch(1, 24, seed=600 + i, vuln_rate=0.5) for i in range(40)]
            rng = np.random.default_rng(0)
            self.ids = [rng.integers(0, 40, 8) for _ in range(16)]

    def trainer(self, engine, seed=1):
        m, tr = new_trainer(engine, seed, use_cuda_graph=self.mode != "eager")
        arena = D.GraphArena.from_graphs(self.graphs, DEV) if self.mode == "arena" else None

        def step(i):
            if self.mode == "arena":
                return float(tr.step_ids(arena, self.ids[i]))
            b = self.host[i % len(self.host)]
            return float(tr.step(b.to(DEV) if self.mode == "eager" else b))
        return m, tr, step


# ---- 1. resume is exact ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["eager", "graph", "arena"])
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_resume_from_a_checkpoint_continues_the_run(engine, mode, tmp_path):
    k = 3
    w = Workload(mode)
    refs = []
    for _ in range(2):                                      # uninterrupted: 2k steps
        m, tr, step = w.trainer(engine)
        refs.append(([step(i) for i in range(2 * k)], params_of(m)))
    m, tr, step = w.trainer(engine)
    losses = [step(i) for i in range(k)]
    torch.save({"state_dict": m.state_dict(), "optimizer": tr.optimizer.state_dict()}, tmp_path / "ckpt.pt")
    saved = [t.clone() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]
    del m, tr, step
    ckpt = torch.load(tmp_path / "ckpt.pt", weights_only=True)
    m, tr, step = w.trainer(engine, seed=99)               # a NEW module (other initial weights) and trainer
    m.load_state_dict(ckpt["state_dict"])
    tr.optimizer.load_state_dict(ckpt["optimizer"])
    for a, b in zip(saved, (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)):
        assert torch.equal(a, b)                            # the state crossed the file bit-exact
    losses += [step(i) for i in range(k, 2 * k)]
    assert_runs_match((losses, params_of(m)), refs[0], refs[1], f"resume {engine} {mode}")


# ---- 2. a load reaches graphs captured before it ----------------------------------------------------------------------
def test_load_into_a_trainer_whose_step_is_already_captured():
    batches = [b.to(DEV) for b in host_batches(2)]
    src_m, src = new_trainer(seed=3)
    for i in range(3):
        src.step(batches[i % 2])
    ckpt = copy.deepcopy({"state_dict": src_m.state_dict(), "optimizer": src.optimizer.state_dict()})

    m, tr = new_trainer(seed=5, use_cuda_graph=True)
    for b in (batches[0], batches[0], batches[1], batches[1]):      # warm-up, capture + replay, capture + replay, replay
        tr.step(b)
    graphs = {k: v[0] for k, v in tr._graphs.items()}
    assert len(graphs) == 2
    m.load_state_dict(ckpt["state_dict"])
    tr.optimizer.load_state_dict(ckpt["optimizer"])
    got = ([float(tr.step(batches[i % 2])) for i in range(4)], params_of(m))
    assert {k: v[0] for k, v in tr._graphs.items()} == graphs      # replays of the graphs captured before the load
    refs = []
    for _ in range(2):                                       # fresh trainers that loaded the same checkpoint
        m2, tr2 = new_trainer(seed=7, use_cuda_graph=True)
        m2.load_state_dict(ckpt["state_dict"])
        tr2.optimizer.load_state_dict(ckpt["optimizer"])
        refs.append(([float(tr2.step(batches[i % 2])) for i in range(4)], params_of(m2)))
    assert_runs_match(got, refs[0], refs[1], "load after capture")


# ---- 3. torch.optim.Adam <-> FusedTrainer ---------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_hand_over_between_torch_adam_and_the_fused_trainer(engine):
    k = 3
    batches = [b.to(DEV) for b in host_batches(2 * k, seed=720)]
    tol = 5e-5 if engine == "simt" else 5e-4                 # test_parity_gpu.py's bounds for the two optimizers
    # torch -> fused: k steps of the reference-style loop, then the fused trainer continues from opt.state_dict()
    m = new_module(engine, seed=2)
    opt = m.configure_optimizers()
    for b in batches[:k]:
        opt.zero_grad()
        m.training_step((b, {}), 0).backward()
        opt.step()
    ckpt = copy.deepcopy({"state_dict": m.state_dict(), "optimizer": opt.state_dict()})
    lt = []
    for b in batches[k:]:
        opt.zero_grad()
        loss = m.training_step((b, {}), 0)
        loss.backward()
        opt.step()
        lt.append(float(loss.detach()))
    mf, trf = new_trainer(engine, seed=4)
    mf.load_state_dict(ckpt["state_dict"])
    trf.optimizer.load_state_dict(ckpt["optimizer"])
    lf = [float(trf.step(b)) for b in batches[k:]]
    assert lf == pytest.approx(lt, abs=5e-5)
    worst_tf = max(float((p - q).abs().max()) for p, q in zip(mf.parameters(), m.parameters()))
    # fused -> torch: torch.optim.Adam takes the fused trainer's state bit-exact and both continue
    sd = trf.optimizer.state_dict()
    mt = new_module(engine, seed=6)
    mt.load_state_dict(mf.state_dict())
    opt2 = torch.optim.Adam(mt.parameters(), lr=1e-3, weight_decay=1e-2)
    opt2.load_state_dict(sd)
    offs = dict(zip(map(id, mf.param_list()), flat_offsets(mf.param_list())[0]))
    for p, q in zip(mt.parameters(), mf.parameters()):
        st, o, n = opt2.state[p], offs[id(q)], q.numel()
        assert int(st["step"]) == 2 * k
        assert torch.equal(st["exp_avg"].reshape(-1), trf.exp_avg[o:o + n])
        assert torch.equal(st["exp_avg_sq"].reshape(-1), trf.exp_avg_sq[o:o + n])
    lf2 = [float(trf.step(b)) for b in batches[:k]]
    lt2 = []
    for b in batches[:k]:
        opt2.zero_grad()
        loss = mt.training_step((b, {}), 0)
        loss.backward()
        opt2.step()
        lt2.append(float(loss.detach()))
    assert lt2 == pytest.approx(lf2, abs=5e-5)
    worst_ft = max(float((p - q).abs().max()) for p, q in zip(mf.parameters(), mt.parameters()))
    print(f"hand-over {engine}: torch->fused max|dparam| {worst_tf:.2e}, fused->torch {worst_ft:.2e}")
    assert worst_tf < tol and worst_ft < tol


def test_reference_checkpoint_next_step_is_reproduced():
    """tests/golden/reference_optimizer_golden.pt: the reference's own module after a few torch.optim.Adam steps, its
    optimizer state, the next batch and the parameters after one more reference step."""
    from deepdfa_b200.batched_graph import BatchedCFG
    fx = torch.load(GOLDEN, weights_only=False)
    m = D.FlowGNNGGNNModule(**fx["ctor"], engine="simt")
    m.load_state_dict(fx["state_dict"])
    m.to(DEV)
    tr = D.FusedTrainer(m)
    tr.optimizer.load_state_dict(fx["optimizer"])           # lr / weight_decay come from the checkpoint's group
    assert tr.lr == fx["lr"] and tr.weight_decay == fx["weight_decay"]
    g = fx["next_graph"]
    loss = float(tr.step(BatchedCFG(g["src"], g["dst"], g["batch_num_nodes"], g["ndata"])))
    worst = max(float((m.state_dict()[k].cpu() - v).abs().max()) for k, v in fx["state_after"].items())
    print(f"reference checkpoint, next step: |dloss| {abs(loss - fx['loss_next']):.2e}, max|dparam| {worst:.2e}")
    assert abs(loss - fx["loss_next"]) < 2e-5
    assert worst < 2e-5


# ---- 4. schedules under CUDA graphs -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lambda", "step"])
def test_lr_schedule_reaches_captured_steps(kind):
    batches = host_batches(3)
    runs = {}
    for mode in ("eager", "eager_again", "graph"):
        m, tr = new_trainer(use_cuda_graph=mode == "graph")
        if kind == "lambda":
            sched = torch.optim.lr_scheduler.LambdaLR(tr.optimizer, lambda s: min(1.0, (s + 1) / 4) * 0.8 ** max(0, s - 4))
        else:
            sched = torch.optim.lr_scheduler.StepLR(tr.optimizer, step_size=2, gamma=0.5)
        losses = []
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            for i in range(9):
                losses.append(float(tr.step(batches[i % 3] if mode == "graph" else batches[i % 3].to(DEV))))
                sched.step()
        sched_warnings = [str(w.message) for w in caught if "lr_scheduler" in str(w.message) or "optimizer.step" in str(w.message)]
        assert not sched_warnings, sched_warnings
        assert tr.lr != 1e-3 and tr.lr == sched.get_last_lr()[0]
        if mode == "graph":
            assert all(st["graph"] is not None for slot in tr._stream_slots.values() for st in slot["sets"])
        runs[mode] = (losses, params_of(m))
    assert_runs_match(runs["graph"], runs["eager"], runs["eager_again"], f"{kind} schedule, graph vs eager")


def test_zero_lr_after_capture_freezes_the_parameters():
    b = host_batches(1)[0].to(DEV)
    m, tr = new_trainer(use_cuda_graph=True)
    for _ in range(3):
        tr.step(b)
    assert len(tr._graphs) == 1
    p0, m0, t0 = tr.flat_p.clone(), tr.exp_avg.clone(), int(tr.step_count)
    tr.optimizer.param_groups[0]["lr"] = 0.0
    for _ in range(2):
        tr.step(b)
    torch.cuda.synchronize()
    assert torch.equal(tr.flat_p, p0)                      # replayed with lr = 0: the update is exactly zero
    assert int(tr.step_count) == t0 + 2 and not torch.equal(tr.exp_avg, m0)     # ... while Adam's state moved on
    tr.lr = 1e-3
    tr.step(b)
    assert not torch.equal(tr.flat_p, p0)


def test_lr_changing_every_step_while_the_host_runs_ahead():
    graphs = [synth.make_batch(1, 24, seed=600 + i, vuln_rate=0.5) for i in range(40)]
    rng = np.random.default_rng(1)
    id_lists = [rng.integers(0, 40, 8) for _ in range(24)]
    runs = {}
    for mode in ("synced", "synced_again", "run_ahead"):
        m, tr = new_trainer(use_cuda_graph=True)
        arena = D.GraphArena.from_graphs(graphs, DEV)
        hist = torch.zeros(len(id_lists), device=DEV)
        for i, ids in enumerate(id_lists):
            tr.lr = 1e-3 * (1 + i % 5) / 3                   # a new value every step, pushed by value in stream order
            hist[i:i + 1].copy_(tr.step_ids(arena, ids))     # no host sync in the run-ahead mode
            if mode != "run_ahead":
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        runs[mode] = (hist.cpu().tolist(), params_of(m))
    assert_runs_match(runs["run_ahead"], runs["synced"], runs["synced_again"], "per-step lr, host running ahead")


# ---- 5. the _hp entry points ----------------------------------------------------------------------------------------
def test_adam_flat_hp_is_bit_identical_and_read_at_run_time():
    torch.manual_seed(0)
    n = 10007
    p0 = torch.randn(n, device=DEV)
    a = [p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)]
    b = [t.clone() for t in a]
    hyper = torch.zeros(5, device=DEV)
    L = lib()
    hps = [(1e-3, 0.9, 0.999, 1e-8, 1e-2), (3e-4, 0.8, 0.99, 1e-6, 0.0), (2e-3, 0.95, 0.9995, 1e-8, 5e-2), (0.0, 0.9, 0.999, 1e-8, 1e-2)]
    for i, hp in enumerate(hps * 2):
        g = torch.randn(n, device=DEV) * (0.1 if i % 2 else 3.0)
        L.call("ddfa_adam_flat", _p(a[0]), _p(g), _p(a[1]), _p(a[2]), _p(a[3]), n, *hp, _stream_ptr())
        hyper.copy_(torch.tensor(hp, dtype=torch.float32))
        L.call("ddfa_adam_flat_hp", _p(b[0]), _p(g), _p(b[1]), _p(b[2]), _p(b[3]), n, _p(hyper), _stream_ptr())
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # a captured launch reads the word at every replay
    g = torch.randn(n, device=DEV)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=s):
            L.call("ddfa_adam_flat_hp", _p(b[0]), _p(g), _p(b[1]), _p(b[2]), _p(b[3]), n, _p(hyper), _stream_ptr())
    torch.cuda.current_stream().wait_stream(s)
    for hp in hps:
        L.call("ddfa_adam_flat", _p(a[0]), _p(g), _p(a[1]), _p(a[2]), _p(a[3]), n, *hp, _stream_ptr())
        hyper.copy_(torch.tensor(hp, dtype=torch.float32))
        graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert int(b[3]) == 2 * len(hps) + len(hps)
    with pytest.raises(D.DdfaError):
        L.call("ddfa_adam_flat_hp", _p(b[0]), _p(g), _p(b[1]), _p(b[2]), _p(b[3]), n, None, _stream_ptr())


@pytest.mark.parametrize("world", [1, 2, 4])
def test_allreduce_adam_p2p_hp_is_bit_identical_and_owner_slices_rebuild_the_moments(world):
    """The one-device emulation of test_allreduce_adam_p2p_protocol_on_one_device, run twice on separate buffer sets — by
    value and through the hyperparameter word — with the same gradients."""
    torch.manual_seed(10 + world)
    n = 64 * 97
    p0 = torch.randn(n, device=DEV)

    def buffers():
        return {"params": [p0.clone() for _ in range(world)], "grads": [torch.zeros(n + 64, device=DEV) for _ in range(world)],
                "flags": [torch.zeros(64, dtype=torch.int32, device=DEV) for _ in range(world)],
                "m": [torch.zeros(n, device=DEV) for _ in range(world)], "v": [torch.zeros(n, device=DEV) for _ in range(world)],
                "step": [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)],
                "ticket": [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)],
                "loss": [torch.zeros(1, device=DEV) for _ in range(world)]}
    sets = {"value": buffers(), "hp": buffers()}
    hyper = [torch.zeros(5, device=DEV) for _ in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    L = lib()
    hps = [(1e-3, 0.9, 0.999, 1e-8, 1e-2), (5e-4, 0.85, 0.995, 1e-7, 3e-2), (2e-3, 0.9, 0.999, 1e-8, 0.0)]
    for it, hp in enumerate(hps):
        gs = [torch.randn(n, device=DEV) * 0.1 for _ in range(world)]
        for key, bs in sets.items():
            for r in range(world):
                bs["grads"][r][:n].copy_(gs[r])
                bs["grads"][r][n] = float(r + 1 + it)
            for h in hyper:
                h.copy_(torch.tensor(hp, dtype=torch.float32))
            torch.cuda.synchronize()
            pp, pg, pf = (ptr_array([_p(t) for t in bs[k]]) for k in ("params", "grads", "flags"))
            for r in range(world):
                common = (pp, pg, pf, r, world, _p(bs["m"][r]), _p(bs["v"][r]), _p(bs["step"][r]), n, n, _p(bs["loss"][r]), _p(bs["ticket"][r]))
                if key == "value":
                    L.call("ddfa_allreduce_adam_p2p", *common, *hp, streams[r].cuda_stream)
                else:
                    L.call("ddfa_allreduce_adam_p2p_hp", *common, _p(hyper[r]), streams[r].cuda_stream)
            torch.cuda.synchronize()
    for k in sets["value"]:
        if k != "flags":
            assert all(torch.equal(x, y) for x, y in zip(sets["value"][k], sets["hp"][k])), k
    # each rank touched exactly its owned_range of the moments; the owners' slices rebuild the full state
    bs = sets["hp"]
    full_m, full_v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    for r in range(world):
        lo, hi = owned_range(n, r, world)
        mask = torch.zeros(n, dtype=torch.bool, device=DEV)
        mask[lo:hi] = True
        assert torch.equal(bs["v"][r] != 0, mask), r         # v > 0 wherever the kernel ran: the helper mirrors the kernel
        full_m[lo:hi] = bs["m"][r][lo:hi]
        full_v[lo:hi] = bs["v"][r][lo:hi]
    for r in range(world):
        lo, hi = owned_range(n, r, world)
        assert torch.equal(full_m[lo:hi], bs["m"][r][lo:hi]) and torch.equal(full_v[lo:hi], bs["v"][r][lo:hi])
    assert bool((full_v > 0).all())


# ---- 6. two GPUs, exchange="p2p" --------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _two_rank_worker(rank, port, q):
    """Both ranks make exactly the same sequence of collective calls (constructors, steps, state_dict); nothing is asserted
    here, so no rank can leave its peer waiting in the p2p kernel.  Results go to the parent as CPU tensors."""
    import torch.distributed as dist
    from deepdfa_b200.batched_graph import split_batch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    out = {}
    try:
        full = [synth.make_batch(32, 40, seed=800 + i, vuln_rate=0.3) for i in range(4)]
        shards = [split_batch(b, 2)[rank].to(dev) for b in full]
        cpu = lambda ts: [t.detach().cpu() for t in ts]     # noqa: E731
        for name in ("A", "A_again"):                        # uninterrupted, 4 steps
            m, tr = new_trainer(seed=1, device=dev, exchange="p2p")
            out[name] = ([float(tr.step(shards[i], global_batch=32)) for i in range(4)], cpu(m.parameters()))
        m, tr = new_trainer(seed=1, device=dev, exchange="p2p")
        losses = [float(tr.step(shards[i], global_batch=32)) for i in range(2)]
        sd = tr.optimizer.state_dict()                       # collective
        msd = {k: v.detach().clone() for k, v in m.state_dict().items()}
        out["state"] = {i: (float(s["step"]), s["exp_avg"].cpu(), s["exp_avg_sq"].cpu()) for i, s in sd["state"].items()}
        m2, tr2 = new_trainer(seed=9, device=dev, exchange="p2p")
        m2.load_state_dict(msd)
        tr2.optimizer.load_state_dict(sd)
        losses += [float(tr2.step(shards[i], global_batch=32)) for i in range(2, 4)]
        out["resumed"] = (losses, cpu(m2.parameters()))
        if rank == 0:                                        # world-2 checkpoint into a world-1 trainer (no collectives)
            m1, tr1 = new_trainer(seed=11, device=dev, distributed=False, exchange="nccl")
            m1.load_state_dict(msd)
            tr1.optimizer.load_state_dict(sd)
            out["world1_loaded"] = [(float(s["step"]), s["exp_avg"].cpu(), s["exp_avg_sq"].cpu())
                                    for s in tr1.optimizer.state_dict()["state"].values()]
            out["world1"] = ([float(tr1.step(full[i].to(dev))) for i in range(2, 4)], cpu(m1.parameters()))
        torch.cuda.synchronize()
        q.put((rank, out))
    except BaseException as exc:                             # reported to the parent, which fails the test
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


def test_two_ranks_p2p_state_dict_and_resume():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, port, q)) for r in range(2)]
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
    r0, r1 = results[0], results[1]
    assert sorted(r0["state"]) == sorted(r1["state"])
    for i, (s0, s1) in enumerate(zip(r0["state"].values(), r1["state"].values())):
        assert s0[0] == s1[0] == 2.0 and torch.equal(s0[1], s1[1]) and torch.equal(s0[2], s1[2]), i     # every rank: the full state
    for s, w in zip(r0["state"].values(), r0["world1_loaded"]):
        assert s[0] == w[0] and torch.equal(s[1], w[1]) and torch.equal(s[2], w[2])
    for r in (r0, r1):
        assert_runs_match(r["resumed"], r["A"], r["A_again"], "two ranks, resumed")
    # the world-1 trainer sums the whole batch's gradient in another order than the two shards do
    dp = max(float((a - b).abs().max()) for a, b in zip(r0["world1"][1], r0["resumed"][1]))
    print(f"world-2 checkpoint continued at world 1: max|dparam| vs world 2 {dp:.2e}")
    assert dp < 5e-4
    assert r0["world1"][0] == pytest.approx(r0["resumed"][0][2:], abs=1e-5)
