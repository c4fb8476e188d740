"""CPU: the shapes of tests/test_scale_gpu.py still reach what those tests are written for — the trip counts of the persistent
tensor-core kernels (csrc/gru_tc_bwd.cu, csrc/gru_tc_fwd3.cu launch formulas) and the hub degrees of the edge gathers.  Fails
if a shape is shrunk below its purpose."""
import numpy as np
import pytest

from deepdfa_b200 import synth
from scale_batches import (GATE_BWD_STAGES, GROUP_IN, HUB_SHAPES, MODULE_C1, OUT_HUB, WGRAD_MAX_STEPS, ZERO_IN, ZERO_OUT, degrees, hub_batch,
                           trip_counts)


@pytest.mark.parametrize("name", list(HUB_SHAPES))
def test_hub_batch_degrees(name):
    g = hub_batch(name)
    N = g.num_nodes()
    src, dst = [t.numpy() for t in g.edges()]
    deg_in, deg_out = degrees(g)
    assert N % 4 and N % 32 and N % 128 and N == HUB_SHAPES[name][2]
    assert {33, 64, 65, 200} <= set(deg_in.tolist()) and deg_in.max() >= 1000
    assert deg_in[N - 1] >= 1000                                     # the last row, inside a ragged last tile, is a hub
    # four consecutive hub rows inside one 4-row warp group (all four above 16, together well above 32 and above 64)
    quads = deg_in[: N // 4 * 4].reshape(-1, 4)
    assert ((quads.min(1) >= min(GROUP_IN)) & (quads.sum(1) > 64)).any()
    assert (deg_out >= 8).sum() >= 10 and deg_out.max() >= OUT_HUB[1]
    off = N - int(g.batch_num_nodes()[-1])
    assert all(deg_in[off + r] == 0 for r in ZERO_IN) and not np.isin(np.array(ZERO_IN) + off, src[src == dst]).any()
    assert all(deg_out[off + r] == 0 for r in ZERO_OUT)
    assert len(np.unique(src.astype(np.int64) * N + dst)) < len(src)    # duplicate edges
    assert int(src.min()) >= 0 and int(max(src.max(), dst.max())) < N


@pytest.mark.parametrize("name,steps", [("threshold", 1), ("c1", 1), ("mid", 8), ("mid", 17)])
def test_kernel_trip_counts(name, steps):
    N = HUB_SHAPES[name][2]
    tc = trip_counts(N, steps)
    assert tc["gate_bwd_blocks"][1] > GATE_BWD_STAGES                 # some gate-backward CTA refills a stage of its ring
    assert tc["gemm_tiles"][0] >= 3                                   # every fwd3 / dgrad3 CTA runs 3 or more tiles
    if name == "threshold":
        assert tc["gate_bwd_blocks"] == (3, 4)                        # just past the threshold: CTAs 0-3 refill exactly once
    if name == "c1":
        assert tc["gate_bwd_blocks"][0] >= 37 and tc["gemm_tiles"][0] >= 37 and tc["wgrad_tiles"][0] > 16
    if steps > 1 and steps <= WGRAD_MAX_STEPS:
        assert tc["wgrad_tiles"][0] > 100                             # the batched weight gradient over all steps
    if steps > WGRAD_MAX_STEPS:
        assert tc["wgrad_tiles"][0] > 10                              # per step, deferred over 17 launches


def test_module_c1_batch_trip_counts():
    g = synth.make_batch(**MODULE_C1)                                 # test_scale_gpu.py::test_module_gradients_at_c1
    tc = trip_counts(g.num_nodes(), 8)
    assert g.num_nodes() > 150_000 and int(g.batch_num_nodes().max()) > 512
    assert tc["gate_bwd_blocks"][0] >= 37 and tc["gemm_tiles"][0] >= 37 and tc["wgrad_tiles"][0] > 400
