"""GPU: the gradient guard — gradient-norm clipping and skipping of non-finite steps inside the fused optimizer step.

Checked: ddfa_grad_norm against fp64 (sizes 0 .. 2^24 + 4, magnitudes 1e-30 .. 1e19, non-finite values at the ends and the
middle), repeatable and equal in both tuning modes; the guarded Adam against clip_grad_norm_ + torch.optim.Adam, bit-identical
to ddfa_adam_flat_hp at coef == 1, and a skipped step that changes nothing; the guarded peer-memory protocol with 1 / 2 / 4 ranks
emulated on one device through a skipped launch; and the trainer: launches with the guard off, bit-identity with an unguarded
run at max_grad_norm = inf, bounds set after capture, the reference loop with clipping, and recovery from a NaN step."""
import contextlib
import math
import os
import socket

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200._lib import lib, ptr_array
from deepdfa_b200.engine import _p, _stream_ptr
from deepdfa_b200.trainer import flat_offsets

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


def module(engine="tcgen05", seed=1, steps=8, device=DEV):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, steps, 2, concat_all_absdf=True, positive_weight=2.0, engine=engine).to(device)


def c1_numel():
    return flat_offsets(module().param_list())[1]


def grad_norm(g, max_norm=None):
    """(gstate[3] on the host, the call's device tensors)."""
    L = lib()
    ws = torch.empty(L.call("ddfa_grad_norm_workspace_bytes", g.numel()), dtype=torch.uint8, device=DEV)
    gstate = torch.full((4,), 7.0, device=DEV)
    mx = None if max_norm is None else torch.full((1,), float(max_norm), device=DEV)
    L.call("ddfa_grad_norm", _p(g) if g.numel() else None, g.numel(), _p(mx), _p(gstate), _p(ws), ws.numel(), _stream_ptr())
    torch.cuda.synchronize()
    return gstate[:3].cpu()


def torch_coef(norm: torch.Tensor, max_norm: float) -> torch.Tensor:
    """clip_grad_norm_'s coefficient from an fp32 norm: clamp(max_norm / (norm + 1e-6), max=1) in fp32."""
    return torch.clamp(torch.tensor(max_norm, dtype=torch.float32) / (norm.reshape(1) + 1e-6), max=1.0)


# ---- 1. the norm --------------------------------------------------------------------------------------------------------
def mixed(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 19, n)
    if n >= 4:
        x[: 4] = [1e-30, -1e19, 1e19, 3.0]
    return torch.from_numpy(x.astype(np.float32)).to(DEV)


@pytest.mark.parametrize("n", [0, 1, 4, 64 * 97, "c1", 2 ** 24 + 4])
def test_grad_norm_matches_fp64_and_is_repeatable(n):
    n = c1_numel() if n == "c1" else n
    g = mixed(n, seed=n)
    ref = math.sqrt(float((g.double() ** 2).sum()))
    with det_mode(False):
        _lib.apply_deterministic_mode()
        a, b = grad_norm(g, 1.0), grad_norm(g, 1.0)
    with det_mode(True):
        _lib.apply_deterministic_mode()
        c = grad_norm(g, 1.0)
    assert torch.equal(a, b) and torch.equal(a, c)          # bit-identical across calls and tuning modes
    norm = float(a[0])
    assert math.isfinite(norm) and a[2] == 0.0
    assert abs(norm - ref) <= 1.2e-7 * ref, (n, norm, ref)
    assert torch.equal(a[1:2], torch_coef(a[0], 1.0))
    # measuring only: no bound (NULL) and +inf both give coef 1
    assert float(grad_norm(g)[1]) == 1.0 and float(grad_norm(g, float("inf"))[1]) == 1.0


@pytest.mark.parametrize("n", [4, 64 * 97, "c1"])
@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_grad_norm_flags_non_finite_values_anywhere(n, bad):
    n = c1_numel() if n == "c1" else n
    for pos in (0, n // 2, n - 1):
        g = torch.randn(n, device=DEV)
        g[pos] = bad
        st = grad_norm(g, 1.0)
        assert st[2] == 1.0 and not math.isfinite(float(st[0])), (n, pos, bad)


# ---- 2. guarded Adam ------------------------------------------------------------------------------------------------------
HP = (1e-3, 0.9, 0.999, 1e-8, 1e-2)


def guarded_step(p, g, m, v, step, max_norm, skipped=None):
    L = lib()
    ws = torch.empty(L.call("ddfa_grad_norm_workspace_bytes", g.numel()), dtype=torch.uint8, device=DEV)
    gstate = torch.zeros(4, device=DEV)
    mx = torch.full((1,), float(max_norm), device=DEV)
    hyper = torch.tensor(HP, device=DEV)
    L.call("ddfa_grad_norm", _p(g), g.numel(), _p(mx), _p(gstate), _p(ws), ws.numel(), _stream_ptr())
    L.call("ddfa_adam_flat_guarded", _p(p), _p(g), _p(m), _p(v), _p(step), p.numel(), _p(hyper), _p(gstate), _p(skipped), _stream_ptr())
    return gstate


def test_guarded_adam_clips_like_torch():
    torch.manual_seed(0)
    n = 10007
    p0 = torch.randn(n)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref], lr=1e-3, weight_decay=1e-2)
    p, m, v = p0.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    for i in range(6):
        g = torch.randn(n) * (0.1 if i % 2 else 3.0)
        ref.grad = g.clone()
        total = torch.nn.utils.clip_grad_norm_([ref], 2.0)
        opt.step()
        st = guarded_step(p, g.to(DEV), m, v, step, 2.0)
        assert float(st[1]) < 1.0 and abs(float(st[0]) - float(total)) <= 1e-6 * float(total)
    assert int(step) == 6
    assert (p.cpu() - ref.detach()).abs().max() < 2e-6


def test_guarded_adam_with_coef_one_is_bit_identical_to_adam_flat_hp():
    torch.manual_seed(1)
    n = 64 * 97 + 3
    a = [torch.randn(n, device=DEV), torch.rand(n, device=DEV) * 0.1, torch.rand(n, device=DEV) * 0.01]
    b = [t.clone() for t in a]
    sa, sb = torch.full((1,), 4, dtype=torch.int32, device=DEV), torch.full((1,), 4, dtype=torch.int32, device=DEV)
    hyper = torch.tensor(HP, device=DEV)
    for i in range(3):
        g = torch.randn(n, device=DEV) * 0.01
        lib().call("ddfa_adam_flat_hp", _p(a[0]), _p(g), _p(a[1]), _p(a[2]), _p(sa), n, _p(hyper), _stream_ptr())
        bound = float("inf") if i == 0 else 1e6            # unbounded, then a bound far above the norm: coef == 1
        st = guarded_step(b[0], g, b[1], b[2], sb, bound)
        assert float(st[1]) == 1.0
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert torch.equal(sa, sb)


def test_guarded_adam_skips_a_nan_step_bit_exactly():
    torch.manual_seed(2)
    n = 4099
    p, m, v = torch.randn(n, device=DEV), torch.rand(n, device=DEV), torch.rand(n, device=DEV)
    step = torch.full((1,), 3, dtype=torch.int32, device=DEV)
    skipped = torch.zeros(1, dtype=torch.int32, device=DEV)
    before = [t.clone() for t in (p, m, v, step)]
    g = torch.randn(n, device=DEV)
    g[1234] = float("nan")
    st = guarded_step(p, g, m, v, step, 1.0, skipped)
    torch.cuda.synchronize()
    assert st[2] == 1.0 and int(skipped) == 1
    for x, y in zip(before, (p, m, v, step)):
        assert torch.equal(x, y)
    # without a skip counter a NaN norm is not hidden: it reaches the update, as in torch
    guarded_step(p, g, m, v, step, 1.0)
    torch.cuda.synchronize()
    assert int(step) == 4 and torch.isnan(p).all()


# ---- 3. the guarded peer-memory protocol, ranks emulated on one device ------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4])
def test_guarded_p2p_protocol_skips_and_recovers(world):
    torch.manual_seed(10 + world)
    n = 64 * 97
    max_norm = 2.0
    p0 = torch.randn(n, device=DEV)
    params = [p0.clone() for _ in range(world)]
    grads = [torch.zeros(n + 64, device=DEV) for _ in range(world)]
    flags = [torch.zeros(128, dtype=torch.int32, device=DEV) for _ in range(world)]
    m = [torch.zeros(n, device=DEV) for _ in range(world)]
    v = [torch.zeros(n, device=DEV) for _ in range(world)]
    step = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)]
    skipped = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)]
    gstate = [torch.zeros(4, device=DEV) for _ in range(world)]
    gws = [torch.zeros(lib().call("ddfa_p2p_guard_state_bytes"), dtype=torch.uint8, device=DEV) for _ in range(world)]
    loss_out = [torch.zeros(1, device=DEV) for _ in range(world)]
    hyper = [torch.tensor(HP, device=DEV) for _ in range(world)]
    mx = [torch.full((1,), max_norm, device=DEV) for _ in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref], lr=1e-3, weight_decay=1e-2)
    L = lib()
    pp, pg, pf = ptr_array([_p(t) for t in params]), ptr_array([_p(t) for t in grads]), ptr_array([_p(t) for t in flags])
    for it in range(5):
        gs = [torch.randn(n, device=DEV) * 0.1 for _ in range(world)]
        if it == 2:
            gs[world - 1][n // 3] = float("nan")
        for r in range(world):
            grads[r][:n].copy_(gs[r])
            grads[r][n] = float(r + 1 + it)
        torch.cuda.synchronize()
        for r in range(world):
            L.call("ddfa_allreduce_adam_p2p_guarded", pp, pg, pf, r, world, _p(m[r]), _p(v[r]), _p(step[r]), n, n, _p(loss_out[r]),
                   _p(hyper[r]), _p(mx[r]), _p(gstate[r]), _p(skipped[r]), _p(gws[r]), streams[r].cuda_stream)
        torch.cuda.synchronize()
        total = torch.stack(gs).sum(0)
        for r in range(world):
            assert torch.equal(gstate[r][:3].view(torch.int32), gstate[0][:3].view(torch.int32)), (it, r)    # the same norm, coef, decision bits
            assert torch.equal(params[r], params[0])
            assert abs(float(loss_out[r]) - sum(q + 1 + it for q in range(world))) < 1e-5
        if it == 2:
            assert gstate[0][2] == 1.0
        else:
            ref64 = float(total.double().norm())
            assert gstate[0][2] == 0.0 and abs(float(gstate[0][0]) - ref64) <= 1.2e-7 * ref64 and float(gstate[0][1]) < 1.0
            ref.grad = total.clone()
            torch.nn.utils.clip_grad_norm_([ref], max_norm)
            opt.step()
        assert (params[0] - ref.detach()).abs().max() < 2e-6, it
        for r in range(world):
            assert int(step[r]) == it + 1 - (1 if it >= 2 else 0), (it, r, int(step[r]))     # applied steps only
            assert int(skipped[r]) == (1 if it >= 2 else 0)
            assert gws[r][:8].view(torch.int32).tolist() == [0, 0]             # both tickets back to zero
            assert int(gws[r][8:12].view(torch.int32)) == it + 1               # the launch counter the epochs come from


# ---- 4. trainer with the guard off: the same launches as before ------------------------------------------------------------
def test_trainer_without_guard_launches_what_it_did_and_refuses_a_bound():
    b = synth.make_batch(32, 60, seed=5, variable=True, vuln_rate=0.3).to(DEV)
    counts = {}
    for name, kw in (("off", {}), ("on", dict(max_grad_norm=1.0, skip_nonfinite=True))):
        tr = D.FusedTrainer(module(seed=3), **kw)
        tr.step(b)
        torch.cuda.synchronize()
        c0 = lib().call("ddfa_launch_count")
        tr.step(b)
        torch.cuda.synchronize()
        counts[name] = lib().call("ddfa_launch_count") - c0
        if name == "off":
            assert tr.max_grad_norm is None and tr.grad_norm is None and tr.skipped_steps == 0
            assert not hasattr(tr, "_gstate") and not tr.ws.scrub_image_tails
            with pytest.raises(ValueError, match="without a gradient guard"):
                tr.max_grad_norm = 1.0
    assert counts["on"] == counts["off"] + 2, counts        # the two norm launches; guarded Adam + its counter replace Adam + its counter


# ---- 5. deterministic mode: max_grad_norm = inf is the unguarded run, bit for bit ----------------------------------------------
def batches(n=3, graphs=256, nodes=150, seed=100):
    return [synth.make_batch(graphs, nodes, seed=seed + i, variable=True, vuln_rate=0.3) for i in range(n)]


def state(tr):
    torch.cuda.synchronize()
    return [t.detach().clone() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]


def assert_same(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("mode", ["eager", "graph", "resident", "arena"])
def test_unbounded_guard_is_bit_identical_to_no_guard(mode):
    bs = batches()
    arena = ids = None
    if mode == "arena":
        graphs = [synth.make_batch(1, 150, seed=3000 + i, vuln_rate=0.5) for i in range(512)]
        arena = D.GraphArena.from_graphs(graphs, DEV)
        rng = np.random.default_rng(0)
        ids = [rng.choice(512, 256, replace=False) for _ in range(3)]
    if mode in ("eager", "resident"):
        bs = [b.to(DEV) for b in bs]
    out = []
    with det_mode():
        for kw in ({}, dict(max_grad_norm=float("inf"), skip_nonfinite=True)):
            tr = D.FusedTrainer(module(seed=7), use_cuda_graph=mode != "eager", **kw)
            losses = []
            for i in range(10):
                losses.append(float(tr.step_ids(arena, ids[i % 3]) if mode == "arena" else tr.step(bs[i % 3])))
            out.append((losses, state(tr)))
            if kw:
                assert tr.skipped_steps == 0 and math.isfinite(float(tr.grad_norm))
    assert out[0][0] == out[1][0]
    assert_same(out[0][1], out[1][1])


def test_bound_changed_after_capture_reaches_the_replay():
    bs = [b.to(DEV) for b in batches(2, graphs=128)]
    runs = []
    with det_mode():
        for graph in (False, True):
            tr = D.FusedTrainer(module(seed=8), use_cuda_graph=graph, max_grad_norm=float("inf"))
            norms = []
            for i in range(8):
                if i == 4:
                    tr.max_grad_norm = 0.5 * norms[-1]          # clips from here on: the captured graphs read the new bound
                tr.step(bs[i % 2])
                norms.append(float(tr.grad_norm))
            runs.append((norms, state(tr)))
            if graph:
                assert len(tr._graphs) == 2
    assert runs[0][0] == runs[1][0]
    assert_same(runs[0][1], runs[1][1])


# ---- 6. clipping against the reference training loop ----------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_clipping_matches_clip_grad_norm_and_torch_adam(engine):
    tol = 5e-5 if engine == "simt" else 5e-4
    bs = [synth.make_batch(16, 40, seed=720 + i, vuln_rate=0.3).to(DEV) for i in range(10)]
    probe = module(engine, seed=2, steps=4)
    probe.training_step((bs[0], {}), 0).backward()
    bound = 0.25 * float(torch.nn.utils.clip_grad_norm_(probe.parameters(), float("inf")))
    m = module(engine, seed=2, steps=4)
    opt = m.configure_optimizers()
    mf = module(engine, seed=2, steps=4)
    mf.load_state_dict(m.state_dict())
    tr = D.FusedTrainer(mf, max_grad_norm=bound)
    for i, b in enumerate(bs):
        opt.zero_grad()
        m.training_step((b, {}), 0).backward()
        total = float(torch.nn.utils.clip_grad_norm_(m.parameters(), bound))
        opt.step()
        tr.step(b)
        assert total > bound, (i, total, bound)                       # every step clips
        if i == 0:
            assert abs(float(tr.grad_norm) - total) <= 1e-4 * total, (float(tr.grad_norm), total)
    worst = max(float((p - q).abs().max()) for p, q in zip(mf.parameters(), m.parameters()))
    print(f"clipping {engine}: max|dparam| {worst:.2e}")
    assert worst < tol


# ---- 7. a NaN step is skipped and leaves nothing behind ---------------------------------------------------------------------
def test_nan_step_is_skipped_and_the_run_continues_as_if_it_never_happened():
    big = synth.make_batch(96, 150, seed=41, variable=True, vuln_rate=0.3).to(DEV)
    small = [synth.make_batch(40, 90, seed=50 + i, variable=True, vuln_rate=0.3).to(DEV) for i in range(4)]
    assert small[0].num_nodes() % 128 and small[0].num_nodes() < big.num_nodes() - 128
    runs = {}
    with det_mode():
        for poisoned in (False, True):
            m = module(seed=9)
            tr = D.FusedTrainer(m, skip_nonfinite=True, max_grad_norm=5.0)
            tr.step(big)
            if poisoned:
                table = m.param_list()[0]                     # embedding table 0: row 0 is the index of most nodes
                keep = table.data[0].clone()
                with torch.no_grad():
                    table.data[0] = float("nan")
                tr.step(big)
                torch.cuda.synchronize()
                assert not math.isfinite(float(tr.grad_norm))
                with torch.no_grad():
                    table.data[0] = keep
            for b in small:
                tr.step(b)
            runs[poisoned] = (state(tr), tr.skipped_steps, tr, m)
    (a, skipped_a, _, _), (b, skipped_b, tr, m) = runs[False], runs[True]
    assert skipped_a == 0 and skipped_b == 1
    assert_same(a, b)
    assert int(b[3]) == 5
    sd = tr.optimizer.state_dict()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-2)
    opt.load_state_dict(sd)
    assert all(int(opt.state[p]["step"]) == 5 for p in m.parameters())


# ---- 8. two GPUs: the decision is the same on both ranks ---------------------------------------------------------------------
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
        full = [synth.make_batch(128, 150, seed=900 + i, variable=True, vuln_rate=0.3) for i in range(3)]
        shards = [split_batch(b, 2)[rank].to(dev) for b in full]
        m = module(seed=7, device=dev)
        tr = D.FusedTrainer(m, distributed=True, exchange=exchange, max_grad_norm=1.0, skip_nonfinite=True)
        gstates = []
        for i in range(6):
            keep = None
            if i == 3 and rank == 1:                          # a NaN on one rank only
                keep = m.param_list()[0].data[0].clone()
                with torch.no_grad():
                    m.param_list()[0].data[0] = float("nan")
            tr.step(shards[i % 3], global_batch=128)
            gstates.append(tr._gstate[:3].detach().cpu().clone())
            if keep is not None:
                torch.cuda.synchronize()
                with torch.no_grad():
                    m.param_list()[0].data[0] = keep
        torch.cuda.synchronize()
        q.put((rank, (gstates, tr.skipped_steps, int(tr.step_count), tr.flat_p.detach().cpu(), tr.exchange)))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_ranks_agree_on_norm_and_skip(exchange):
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
    for r in (0, 1):
        assert not isinstance(res[r], str), res[r]
    (g0, s0, c0, p0, e0), (g1, s1, c1, p1, e1) = res[0], res[1]
    assert e0 == e1 == exchange
    for a, b in zip(g0, g1):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))    # norm bits and decision agree (NCCL: equal all-reduced copies)
    assert g0[3][2] == 1.0 and s0 == s1 == 1 and c0 == c1 == 5
    assert torch.equal(p0, p1)
