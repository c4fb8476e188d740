"""Cost of the label_style="node" draw over several ranks at the benchmark's C1 batch, with CUDA events.

    python scripts/node_dp_cost.py [--iters 50] [--steps 20] [--rounds 5]

One GPU: the phased draw of ``engine.NodeDrawDP`` (ddfa_node_dp_*) for R = 1, 2, 4 node-balanced shards of the C1 batch (1024
graphs x 150 nodes), the exchanges between the phases emulated with torch sums and left out of the timing (events around every
phase group), against ``ddfa_node_sample`` on the whole batch.  Per R: the slowest rank's phase time, for factor None and 1.0.

Two or more GPUs: the captured C1 node step (tensor-core engine, NCCL exchange) in ms per rank, R = 1 against R = 2 (each rank
a C1/2 shard), for factor None and 1.0, and the one-rank step on rank 0's shard alone: ``two_rank_overhead_ms`` is what the
second rank adds to a step of the same shard — the draw's collectives (run on a side stream under the GGNN forward) and the
gradient all-reduce.  With a single GPU these rows are reported as not run.  Prints one JSON line with the card's name and
power limit, read in the same run."""
import argparse
import json
import os
import socket
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import engine as E  # noqa: E402
from deepdfa_b200 import synth  # noqa: E402
from deepdfa_b200.batched_graph import partition_graphs, split_batch  # noqa: E402

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def med(xs):
    return sorted(xs)[len(xs) // 2]


class Spans:
    """Sums the device time of the enqueued spans (an event pair each), so the host-side exchanges between them do not count."""

    def __init__(self):
        self.pairs = []

    def __call__(self, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        self.pairs.append((a, b))

    def total(self):
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.pairs)


def phased(vuln, cuts, factor, dev):
    """Per rank a NodeDrawDP over its shard and the (rank -> Spans) of one full draw, exchanges emulated between the phases."""
    R = len(cuts) - 1
    draws = []
    for r in range(R):
        v = vuln[cuts[r]:cuts[r + 1]].contiguous()
        w = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(4)]
        draws.append(E.NodeDrawDP(v, torch.tensor([v.numel()], dtype=torch.int32, device=dev), factor, 7,
                                  torch.zeros(1, dtype=torch.int64, device=dev), torch.empty(v.numel(), dtype=torch.int32, device=dev),
                                  *w, r, R))

    def run():
        spans = [Spans() for _ in range(R)]

        def phase(fn):
            for r, d in enumerate(draws):
                spans[r](lambda: fn(d))

        def exchange(region):
            parts = [region(d) for d in draws]
            total = torch.stack(parts).sum(0).to(torch.int32)
            for p in parts:
                p.copy_(total)
        phase(lambda d: d.count())
        exchange(lambda d: d.counts())
        phase(lambda d: d.plan())
        if factor is not None:
            for p in range(4):
                phase(lambda d: d.radix_hist(p))
                exchange(lambda d: d.hist())
                phase(lambda d: d.radix_pick(p))
            phase(lambda d: d.tie_count())
            exchange(lambda d: d.ties())
            phase(lambda d: d.finish())
        return max(s.total() for s in spans)
    return run


def one_gpu(args, dev):
    g = synth.make_batch(1024, 150, seed=0)
    vuln = g.ndata["_VULN"].to(dev).to(torch.int32).contiguous()
    N = vuln.numel()
    ptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(g.batch_num_nodes(), 0)])
    out = {}
    for factor in (None, 1.0):
        rows = torch.empty(N, dtype=torch.int32, device=dev)
        w = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(3)]
        draw = torch.zeros(1, dtype=torch.int64, device=dev)
        nv = torch.tensor([N], dtype=torch.int32, device=dev)
        ws = E.Workspace(dev)

        def sample():
            E.node_sample(vuln, nv, factor, 7, draw, rows, w[0], w[1], alloc=ws)
        sample()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t1 = []
        for _ in range(args.rounds):
            a.record()
            for _ in range(args.iters):
                sample()
            b.record()
            torch.cuda.synchronize()
            t1.append(a.elapsed_time(b) / args.iters)
        key = "none" if factor is None else f"{factor:g}"
        row = {"ddfa_node_sample_ms": round(med(t1), 4)}
        for R in (1, 2, 4):
            cuts = [int(ptr[o]) for o in partition_graphs(g.batch_num_nodes(), R)]
            run = phased(vuln, cuts, factor, dev)
            run()
            ts = [med([run() for _ in range(args.iters)]) for _ in range(args.rounds)]
            row[f"phased_R{R}_slowest_rank_ms"] = round(med(ts), 4)
        out[f"factor_{key}"] = row
    return out


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _step_ms(tr, batch, steps, rounds):
    for _ in range(3):                      # eager warm-up, capture, replay
        tr.step(batch)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(rounds):
        a.record()
        for _ in range(steps):
            tr.step(batch)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / steps)
    return med(ts)


def _worker(rank, port, args, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_WORLD_SIZE="2")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device(dev))
    try:
        full = synth.make_batch(1024, 150, seed=0)
        shard = split_batch(full, 2)[rank].to(dev)
        half = split_batch(full, 2)[0].to(dev)
        res = {}
        for factor in (None, 1.0):
            torch.manual_seed(0)
            kw = dict(label_style="node", undersample_node_on_loss_factor=factor, positive_weight=2.0, engine="tcgen05")
            m2 = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, **kw).to(dev)
            t2 = _step_ms(D.FusedTrainer(m2, distributed=True, exchange="nccl", use_cuda_graph=True), shard, args.steps, args.rounds)
            dist.barrier()
            m1 = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, **kw).to(dev)
            t1h = _step_ms(D.FusedTrainer(m1, distributed=False, use_cuda_graph=True), half, args.steps, args.rounds)
            m1f = D.FlowGNNGGNNModule(FEAT, 1002, 32, 8, 2, concat_all_absdf=True, **kw).to(dev)
            t1 = _step_ms(D.FusedTrainer(m1f, distributed=False, use_cuda_graph=True), full.to(dev), args.steps, args.rounds)
            key = "none" if factor is None else f"{factor:g}"
            res[f"factor_{key}"] = {"R1_step_ms": round(t1, 3), "R2_step_ms_per_rank": round(t2, 3),
                                    "R1_step_ms_on_the_half_batch": round(t1h, 3)}
        q.put((rank, res))
    except BaseException as exc:
        q.put((rank, f"{type(exc).__name__}: {exc}"))
    finally:
        dist.destroy_process_group()


def two_gpus(args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, args, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=1800) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
    if isinstance(res[0], str) or isinstance(res[1], str):
        return {"error": [res[0], res[1]]}
    out = {}
    for key, r0 in res[0].items():
        r = dict(r0)
        r["R2_step_ms_per_rank"] = max(r0["R2_step_ms_per_rank"], res[1][key]["R2_step_ms_per_rank"])
        # the exposed cost of the two-rank step over a one-rank step on the same shard: the draw's collectives and the gradient
        # all-reduce; "hidden" when it is below the draw's own one-GPU time would suggest (the collectives sit under the forward)
        r["two_rank_overhead_ms"] = round(r["R2_step_ms_per_rank"] - r0["R1_step_ms_on_the_half_batch"], 3)
        out[key] = r
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("node_dp_cost.py measures on the GPU; no CUDA device found")
    result = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "gpus": torch.cuda.device_count(),
              "one_gpu": one_gpu(args, "cuda:0")}
    result["two_gpus"] = two_gpus(args) if torch.cuda.device_count() >= 2 else "not run: one GPU"
    print(json.dumps(result))


if __name__ == "__main__":
    main()
