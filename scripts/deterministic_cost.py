"""Cost of deterministic mode (DDFA_TUNE_DETERMINISTIC) per replaced reduction, at the benchmark's C1 batch, with CUDA events.

    python scripts/deterministic_cost.py [--iters 20]

Times, in both modes, the calls of engine.backward whose reductions change (embedding backward, readout backward, the GRU steps,
the MLP backward, the loss) and the whole forward + backward of the module.  Prints one JSON line per mode."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deepdfa_b200 as D  # noqa: E402
from deepdfa_b200 import _lib, synth  # noqa: E402
from deepdfa_b200 import engine as E  # noqa: E402

TAGS = ("ddfa_embed_concat_bwd", "ddfa_readout_bwd", "ddfa_gru_step_bwd")


class Hook:
    def __init__(self):
        self.ev = {t: [] for t in TAGS}
        self.open = {}

    def wants(self, name):
        return name in self.ev

    def begin(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.open[name] = e

    def end(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.ev[name].append((self.open.pop(name), e))


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deterministic_cost.py measures on the GPU; no CUDA device found")
    dev = "cuda:0"
    torch.manual_seed(0)
    m = D.FlowGNNGGNNModule("_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000", 1002, 32, 8, 2, concat_all_absdf=True,
                            positive_weight=2.0, engine="tcgen05").to(dev)
    batch = synth.make_batch(1024, 150, seed=11, variable=True, vuln_rate=0.3).to(dev)
    L = _lib.lib()
    B, D2 = batch.batch_size, 256
    dlog = torch.randn(B, device=dev)
    pooled = torch.randn(B, D2, device=dev)
    act = torch.relu(torch.randn(1, B, D2, device=dev))
    ws = [torch.randn(D2, D2, device=dev), torch.randn(1, D2, device=dev)]
    gw = [torch.zeros_like(w) for w in ws]
    gb = [torch.zeros(D2, device=dev), torch.zeros(1, device=dev)]
    dpool = torch.empty(B, D2, device=dev)
    scratch = torch.empty(2, B, D2, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    name = torch.cuda.get_device_name()
    for det in (0, 1):
        os.environ["DDFA_DETERMINISTIC"] = str(det)
        _lib.apply_deterministic_mode()

        def step():
            m.zero_grad(set_to_none=True)
            m.training_step((batch, None)).backward()

        def mlp():
            L.call("ddfa_mlp_bwd", dlog.data_ptr(), pooled.data_ptr(), act.data_ptr(), _lib.ptr_array([w.data_ptr() for w in ws]), B, 128, 2,
                   dpool.data_ptr(), _lib.ptr_array([w.data_ptr() for w in gw]), _lib.ptr_array([b.data_ptr() for b in gb]),
                   scratch.data_ptr(), st)
        step_us = timed(step, args.iters)
        mlp_us = timed(mlp, args.iters)
        hook = Hook()
        E.profile_hook = hook
        for _ in range(args.iters):
            step()
        torch.cuda.synchronize()
        E.profile_hook = None
        per = {t: sum(a.elapsed_time(b) for a, b in v) * 1e3 / args.iters for t, v in hook.ev.items()}
        print(json.dumps({"device": name, "deterministic": det, "module_fwd_bwd_us": round(step_us, 1), "mlp_bwd_B1024_us": round(mlp_us, 1),
                          **{f"{t}_us_per_backward": round(v, 1) for t, v in per.items()}}))


if __name__ == "__main__":
    main()
