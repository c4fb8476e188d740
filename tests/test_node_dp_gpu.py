"""GPU: label_style="node" over several ranks — the loss rows drawn over the global batch (the ranks' shards concatenated in rank
order), each rank keeping the rows in its shard.

Part 1 emulates the ranks on one device: the phase entry points (``engine.NodeDrawDP``) of every shard are called in lockstep and
the exchanges between them are torch sums.  The union of ``node_offset + rows`` must be ``ddfa_node_sample`` on the concatenated
batch bit for bit (same S, status and draw), the per-rank dlogits bit-identical to the one-rank rows', and the per-rank loss
shares must sum to the one-rank loss.  Part 2 needs two GPUs: two NCCL ranks of FusedTrainer over ``split_batch`` shards against
one rank over the global batch."""
import os
import socket

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import engine as E, synth
from deepdfa_b200.batched_graph import partition_graphs
from head_batches import c1_batch, tie_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


# ---- 1. emulated ranks on one device -----------------------------------------------------------------------------------------
def one_rank(vuln, factor, seed, draw):
    """ddfa_node_sample over the whole (unpadded) vector: (rows, S, status, next draw)."""
    N = len(vuln)
    v = torch.as_tensor(vuln, dtype=torch.int32, device=DEV)
    nv = torch.tensor([N], dtype=torch.int32, device=DEV)
    rows = torch.empty(max(N, 1), dtype=torch.int32, device=DEV)
    S, status = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    d = torch.tensor([draw], dtype=torch.int64, device=DEV)
    E.node_sample(v, nv, factor, seed, d, rows[:N] if N else rows, S, status)
    torch.cuda.synchronize()
    return rows[:int(S)].cpu(), int(S), int(status), int(d)


def emulated(vuln, cuts, pads, factor, seed, draw):
    """The phased draw of every shard vuln[cuts[r]:cuts[r+1]], padded by pads[r] tail nodes (vulnerable ones among them), with
    the exchanges done by torch sums.  Returns per rank (rows, S_local, S_global, offset, status, next draw) and the draws."""
    R = len(cuts) - 1
    rng = np.random.default_rng(len(vuln) + R)
    draws = []
    for r in range(R):
        local = np.asarray(vuln[cuts[r]:cuts[r + 1]], dtype=np.int32)
        n = len(local)
        pad = (rng.random(pads[r]) < 0.5).astype(np.int32)          # padding nodes: excluded through the valid count
        v = torch.as_tensor(np.concatenate([local, pad]), dtype=torch.int32, device=DEV)
        cap = n + pads[r]
        words = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(5)]
        d = torch.tensor([draw], dtype=torch.int64, device=DEV)
        rows = torch.full((max(cap, 1),), -7, dtype=torch.int32, device=DEV)
        nv = torch.tensor([n], dtype=torch.int32, device=DEV)
        draws.append((E.NodeDrawDP(v, nv, factor, seed, d, rows[:cap] if cap else rows[:0], words[0], words[1], words[2], words[3],
                                   r, R), v, d, words))

    def exchange(region):
        parts = [region(dr) for dr, *_ in draws]
        total = torch.stack(parts).sum(0).to(torch.int32)
        for p in parts:
            p.copy_(total)
    for dr, *_ in draws:
        dr.count()
    exchange(lambda dr: dr.counts())
    for dr, *_ in draws:
        dr.plan()
    if factor is not None:
        for p in range(4):
            for dr, *_ in draws:
                dr.radix_hist(p)
            exchange(lambda dr: dr.hist())
            for dr, *_ in draws:
                dr.radix_pick(p)
        for dr, *_ in draws:
            dr.tie_count()
        exchange(lambda dr: dr.ties())
        for dr, *_ in draws:
            dr.finish()
    torch.cuda.synchronize()
    out = []
    for dr, v, d, (S, status, Sg, off, _) in draws:
        out.append((dr.rows[:int(S)].cpu(), int(S), int(Sg), int(off), int(status), int(d)))
    return out, draws


def c1_cuts(vuln_len, R):
    g = c1_batch()
    offs = partition_graphs(g.batch_num_nodes(), R)
    ptr = np.concatenate([[0], np.cumsum(g.batch_num_nodes().numpy())])
    cuts = [int(ptr[o]) for o in offs]
    assert cuts[0] == 0 and cuts[-1] == vuln_len
    return cuts


def check_union(vuln, cuts, pads, factor, seed, draw):
    ref_rows, ref_S, ref_status, ref_draw = one_rank(vuln, factor, seed, draw)
    got, draws = emulated(vuln, cuts, pads, factor, seed, draw)
    union = torch.cat([rows.long() + off for rows, _, _, off, _, _ in got])
    assert torch.equal(union, ref_rows.long())
    for r, (rows, S, Sg, off, status, d) in enumerate(got):
        assert off == cuts[r] and Sg == ref_S and status == ref_status
        assert d == (ref_draw if factor is not None else draw)
        assert rows.numel() == 0 or (int(rows.min()) >= 0 and int(rows.max()) < cuts[r + 1] - cuts[r])
    assert sum(S for _, S, *_ in got) == ref_S
    return ref_rows, got, draws


@pytest.mark.parametrize("R", [2, 3, 4])
@pytest.mark.parametrize("factor", [None, 1.0, "over"])
def test_emulated_ranks_draw_the_one_rank_rows_of_the_global_batch(R, factor):
    g = c1_batch()
    vuln = g.ndata["_VULN"].numpy().astype(np.int32).copy()
    cuts = c1_cuts(len(vuln), R)
    vuln[cuts[1]:cuts[2]] = 0                     # one shard without a vulnerable node
    pads = [0, 300, 0, 1000][:R]                  # bucket padding at some shards' tails
    f = 1e6 if factor == "over" else factor       # an oversized draw: the whole population, status set on every rank
    _, got, _ = check_union(vuln, cuts, pads, f, seed=11, draw=40)
    if factor == "over":
        assert all(status == 1 for *_, status, _ in got)
    else:
        assert all(status == 0 for *_, status, _ in got)


def test_one_rank_phases_are_ddfa_node_sample():
    g = c1_batch()
    vuln = g.ndata["_VULN"].numpy().astype(np.int32)
    for factor in (None, 0.5, 2.0):
        check_union(vuln, [0, len(vuln)], [0], factor, seed=5, draw=(1 << 32) + 3)


@pytest.mark.parametrize("which", ["factor_a", "factor_ab"])
def test_threshold_ties_straddling_a_rank_boundary(which):
    t = tie_case()
    assert t is not None
    a, b, vuln = t["a"], t["b"], t["vuln"]
    mid = (a + b) // 2 + 1                         # a on rank 0, b on rank 1
    cuts = [0, mid, len(vuln)]
    ref_rows, got, _ = check_union(vuln, cuts, [0, 64], t[which], seed=t["seed"], draw=0)
    assert (a in ref_rows.tolist()) and ((b in ref_rows.tolist()) == (which == "factor_ab"))
    cuts3 = [0, a + 1, b, len(vuln)]              # three ranks: a last on rank 0, b first on rank 2
    check_union(vuln, cuts3, [0, 0, 0], t[which], seed=t["seed"], draw=0)


@pytest.mark.parametrize("R", [2, 4])
@pytest.mark.parametrize("factor", [None, 1.0])
@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
def test_per_rank_bce_is_the_one_rank_bce(R, factor, grad_scale):
    g = c1_batch()
    vuln = g.ndata["_VULN"].numpy().astype(np.int32)
    N = len(vuln)
    cuts = c1_cuts(N, R)
    pads = [0, 200, 0, 17][:R]
    ref_rows, got, draws = check_union(vuln, cuts, pads, factor, seed=9, draw=2)
    node_logit = torch.randn(N, generator=torch.Generator().manual_seed(3)) * 4
    pw = 3.0
    # one rank
    S = len(ref_rows)
    lg = torch.zeros(N, device=DEV)
    lg[:S] = node_logit[ref_rows.long()].to(DEV)
    rows_d = torch.zeros(N, dtype=torch.int32, device=DEV)
    rows_d[:S] = ref_rows.to(DEV)
    S_d = torch.tensor([S], dtype=torch.int32, device=DEV)
    loss1 = torch.zeros(1, device=DEV)
    v_d = torch.as_tensor(vuln, dtype=torch.int32, device=DEV)
    if grad_scale == 1.0:
        dl1 = E.node_bce(lg, v_d, rows_d, S_d, pw, loss1).clone()
    else:
        dl1 = E.node_bce(lg, v_d, rows_d, S_d, pw, loss1, grad_scale=grad_scale).clone()
    # every rank
    shares, dls = [], []
    for r, (dr, v, _, words) in enumerate(draws):
        cap = dr.N
        lr_ = torch.zeros(max(cap, 1), device=DEV)
        rows_r, S_r = got[r][0], got[r][1]
        lr_[:S_r] = node_logit[rows_r.long() + cuts[r]].to(DEV)
        loss_r = torch.zeros(1, device=DEV)
        dl = E.node_bce_global(lr_, v, dr.rows if cap else torch.zeros(1, dtype=torch.int32, device=DEV), dr.num_rows,
                               dr.num_rows_global, pw, loss_r, grad_scale=grad_scale)
        torch.cuda.synchronize()
        shares.append(float(loss_r))
        dls.append(dl[:S_r].cpu())
    assert torch.equal(torch.cat(dls), dl1[:S].cpu())
    total, ref = sum(shares), float(loss1)
    assert abs(total - ref) <= 1e-6 * abs(ref), (total, ref)


# ---- 2. two NCCL ranks ---------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def node_module(factor, device, seed=7):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, label_style="node", concat_all_absdf=True, engine="simt",
                               undersample_node_on_loss_factor=factor, positive_weight=2.0).to(device)


def _compare(rank, dev, factor, mode, exchange, steps=5, **kw):
    """2-rank trainer over split_batch shards against the 1-rank trainer over the global batch: per step the mapped rows and
    the losses, then the largest parameter difference.  mode: "eager" (device batches), "resident" (device batch objects,
    captured) or "bucket" (host batches padded to bucket shapes, captured).  Two batches alternate, so captured graphs replay."""
    from deepdfa_b200.batched_graph import split_batch
    full = [synth.make_batch(48, 60, seed=700 + i, variable=True, vuln_rate=0.3) for i in range(2)]
    host = mode == "bucket"
    shards = [split_batch(b, 2)[rank] for b in full]
    shards, full = (shards, full) if host else ([s.to(dev) for s in shards], [b.to(dev) for b in full])
    if host:
        kw.update(bucket_nodes=1024, bucket_edges=4096)
    m2, m1 = node_module(factor, dev), node_module(factor, dev)
    t2 = D.FusedTrainer(m2, distributed=True, exchange=exchange, use_cuda_graph=mode != "eager", node_sample_seed=5, **kw)
    t1 = D.FusedTrainer(m1, distributed=False, use_cuda_graph=mode != "eager", node_sample_seed=5, **kw)
    rows_ok, dloss = True, 0.0
    for i in range(steps):
        b, shard = full[i % 2], shards[i % 2]
        l2 = float(t2.step(shard))
        l1 = float(t1.step(b))
        off, r1 = t2.last_node_offset(), t1.last_loss_rows().long()
        mine = r1[(r1 >= off) & (r1 < off + shard.num_nodes())] - off
        rows_ok &= torch.equal(t2.last_loss_rows().long(), mine) and t2.last_num_rows_global() == r1.numel()
        if kw.get("accumulate_grad_batches", 1) == 1:
            dloss = max(dloss, abs(l2 - l1) / max(1.0, abs(l1)))
    torch.cuda.synchronize()
    dparam = max(float((p.data - q.data).abs().max()) for p, q in zip(m2.param_list(), m1.param_list()))
    return rows_ok, dloss, dparam, t2.exchange


def _compare_arena(rank, dev, exchange):
    """step_ids over a GraphArena: rank r trains on its half of each id list (captured), one rank on the whole list."""
    graphs = [synth.make_batch(1, 40, seed=600 + i, vuln_rate=0.3) for i in range(40)]
    arena = D.GraphArena.from_graphs(graphs, dev)
    m2, m1 = node_module(1.0, dev), node_module(1.0, dev)
    t2 = D.FusedTrainer(m2, distributed=True, exchange=exchange, use_cuda_graph=True)
    t1 = D.FusedTrainer(m1, distributed=False, use_cuda_graph=True)
    rows_ok, dloss = True, 0.0
    for i in range(5):
        ids = np.random.default_rng(i % 2).integers(0, 40, 16)          # two id lists alternate: captured graphs replay
        half = ids[:8] if rank == 0 else ids[8:]
        l2 = float(t2.step_ids(arena, half))
        l1 = float(t1.step_ids(arena, ids))
        off, r1 = t2.last_node_offset(), t1.last_loss_rows().long()
        n = int(arena.nodes_per_graph[half].sum())
        rows_ok &= torch.equal(t2.last_loss_rows().long(), r1[(r1 >= off) & (r1 < off + n)] - off)
        dloss = max(dloss, abs(l2 - l1) / max(1.0, abs(l1)))
    torch.cuda.synchronize()
    dparam = max(float((p.data - q.data).abs().max()) for p, q in zip(m2.param_list(), m1.param_list()))
    return rows_ok, dloss, dparam, t2.exchange


def _worker(rank, port, exchange, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2", DDFA_DETERMINISTIC="1")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    try:
        res = {}
        for factor in (None, 1.0):
            for mode in ("eager", "resident", "bucket"):
                res[(mode, factor)] = _compare(rank, dev, factor, mode, exchange)
        res["accumulate"] = _compare(rank, dev, 1.0, "bucket", exchange, steps=6, accumulate_grad_batches=2, max_grad_norm=0.5)
        res["arena"] = _compare_arena(rank, dev, exchange)
        for factor in (None, 1.0):
            res[("self_check", factor)] = D.FusedTrainer.dp_self_check("simt", dev, rank, 2, exchange=exchange, label_style="node",
                                                                       factor=factor)
        try:
            D.FusedTrainer(node_module(1.0, dev), distributed=True, exchange=exchange, node_sample_seed=rank)
            res["seed"] = "no error"
        except ValueError as exc:
            res["seed"] = str(exc)
        q.put((rank, res))
    except BaseException as exc:
        import traceback
        q.put((rank, f"{type(exc).__name__}: {exc}\n{traceback.format_exc()}"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_two_ranks_train_node_style_as_one_rank_over_the_global_batch(exchange):
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
            rank, out = q.get(timeout=900)
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
        out = res[r]
        assert not isinstance(out, str), out
        for key, val in out.items():
            if key == "seed":
                assert "node_sample_seed differs" in val, val
            elif key[0] == "self_check":
                assert val["rows_identical"] and val["max_abs_loss_diff"] <= 1e-5 and val["max_abs_param_diff"] <= 1e-3, (key, val)
            else:
                rows_ok, dloss, dparam, used = val
                assert used == exchange, (key, used)
                assert rows_ok, key
                assert dloss <= 1e-5, (key, dloss)
                assert dparam <= 1e-3, (key, dparam)


# ---- 3. the trainer's several-rank path on one device --------------------------------------------------------------------------
@pytest.fixture
def rank0_of_two(monkeypatch):
    """A real one-process NCCL group that the trainer is told is rank 0 of two.  Every SUM over it returns this rank's words,
    which is what two ranks return when rank 1's shard is empty: rank 1 adds zero counts, zero histograms, zero ties and
    zero gradients.  So the several-rank step — side-stream draw, captured collectives, global-S BCE — must reproduce the
    one-rank trainer on the same batch bit for bit."""
    import torch.distributed as dist
    import deepdfa_b200.trainer as T
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1,
                            device_id=torch.device(DEV))
    monkeypatch.setattr(T.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
    try:
        yield
    finally:
        monkeypatch.undo()
        dist.destroy_process_group()


def _pair(factor, mode, **kw):
    full = [synth.make_batch(24, 60, seed=800 + i, variable=True, vuln_rate=0.3) for i in range(2)]
    if mode != "bucket":
        full = [b.to(DEV) for b in full]
    else:
        kw.update(bucket_nodes=1024, bucket_edges=4096)
    out = []
    for distributed in (True, False):
        m = node_module(factor, DEV)
        tr = D.FusedTrainer(m, distributed=distributed, exchange="nccl", use_cuda_graph=mode != "eager", node_sample_seed=3, **kw)
        assert tr.world == (2 if distributed else 1)
        losses, rows, extra = [], [], []
        for i in range(5):
            losses.append(float(tr.step(full[i % 2])))
            rows.append(tr.last_loss_rows().cpu())
            extra.append((tr.last_node_offset(), tr.last_num_rows_global()))
        torch.cuda.synchronize()
        out.append((losses, rows, extra, [p.detach().clone() for p in m.parameters()], tr))
    return out


@pytest.mark.parametrize("mode", ["eager", "resident", "bucket"])
@pytest.mark.parametrize("factor", [None, 1.0])
def test_several_rank_step_with_an_empty_peer_is_the_one_rank_step(rank0_of_two, mode, factor):
    (l2, r2, x2, p2, t2), (l1, r1, x1, p1, _) = _pair(factor, mode)
    assert all(torch.equal(a, b) for a, b in zip(r2, r1))
    assert x2 == [(0, r.numel()) for r in r1] == x1
    assert l2 == l1
    assert all(torch.equal(a, b) for a, b in zip(p2, p1))
    if mode != "eager":
        assert t2._graphs or any(st["graph"] is not None for s in t2._stream_slots.values() for st in s["sets"])


def test_several_rank_step_with_accumulation_and_clipping(rank0_of_two):
    (l2, r2, _, p2, _), (l1, r1, _, p1, _) = _pair(1.0, "bucket", accumulate_grad_batches=2, max_grad_norm=0.5)
    assert all(torch.equal(a, b) for a, b in zip(r2, r1)) and l2 == l1
    assert all(torch.equal(a, b) for a, b in zip(p2, p1))


def test_several_rank_step_ids_over_an_arena(rank0_of_two):
    graphs = [synth.make_batch(1, 40, seed=600 + i, vuln_rate=0.3) for i in range(30)]
    arena = D.GraphArena.from_graphs(graphs, DEV)
    res = []
    for distributed in (True, False):
        m = node_module(1.0, DEV)
        tr = D.FusedTrainer(m, distributed=distributed, exchange="nccl", use_cuda_graph=True, track_metrics=True)
        ls, rs = [], []
        for i in range(5):
            ls.append(float(tr.step_ids(arena, np.random.default_rng(i % 2).integers(0, 30, 8))))
            rs.append(tr.last_loss_rows().cpu())
        res.append((ls, rs, [p.detach().clone() for p in m.parameters()], tr.metrics()))
    (l2, r2, p2, m2), (l1, r1, p1, m1) = res
    assert l2 == l1 and all(torch.equal(a, b) for a, b in zip(r2, r1)) and all(torch.equal(a, b) for a, b in zip(p2, p1))
    assert m2 == m1


def test_oversized_draw_raises_one_step_late_on_several_ranks(rank0_of_two):
    b = synth.make_batch(12, 40, seed=5, variable=True, vuln_rate=0.6).to(DEV)
    tr = D.FusedTrainer(node_module(500.0, DEV), distributed=True, exchange="nccl")
    tr.step(b)
    with pytest.raises(ValueError, match="more non-vulnerable"):
        tr.check_inputs()
