"""GPU: the fused backward GRU step (bwd_step_fused_kernel: gate backward and dgrad in one 4-CTA cluster kernel) against the
two-kernel path it replaces (DDFA_TUNE_GATE_BWD_TMA = 0: gate_bwd_image_kernel, then dgrad3_kernel).

Both paths do the same arithmetic in the same order, so ds, dh and the weight gradients must come out bit-identical; the weight
gradient GEMM is deterministic, so equal dW' / dWhh also means equal q images, padding rows included.  Only the bias gradients
are summed in another order (per-warp column sums, combined through atomics)."""
import ctypes

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import synth
from deepdfa_b200._lib import ENGINE_TCGEN05, TUNE_GATE_BWD_TMA, DdfaError, lib
from deepdfa_b200.engine import _p, _stream_ptr, prepare_graph
from scale_batches import hub_batch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D_ = 128
GRADS = ("dwf", "dbf", "dbih", "dwhh", "dbhh")
BIASES = ("dbf", "dbih", "dbhh")
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


def _batch(case):
    if case == "n_lt_128":
        return synth.make_batch(1, 100, seed=21)                     # one ragged tile
    if case == "tile_plus_1":
        return synth.make_batch(seed=22, sizes=[125] * 40 + [121])        # 128 k + 1 nodes: a last tile of one row
    if case == "few_tiles":
        return synth.make_batch(9, 150, seed=23)                     # 11 tiles: fewer tiles than clusters
    if case == "c0":
        return synth.make_batch(256, 150, 2.0, 1002, seed=24)        # the benchmark's C0 batch shape
    return hub_batch("threshold")                                    # hub rows, 12 701 nodes


@pytest.fixture(scope="module")
def L():
    return lib()


def test_cluster_occupancy(L):
    """The fused kernel runs one CTA per SM in clusters of four: at most 33 resident clusters on a 132-SM H100 (30 measured:
    a cluster has to fit inside one GPC)."""
    v = ctypes.c_int(0)
    L.call("ddfa_debug_read", 5, ctypes.byref(v), 4)
    print(f"bwd_step_fused_kernel: {v.value} clusters of 4 CTAs resident at once")
    assert 1 <= v.value <= 33


@pytest.mark.parametrize("case", ["n_lt_128", "tile_plus_1", "few_tiles", "c0", "hub"])
def test_fused_bwd_matches_two_kernel_path(L, case):
    g = _batch(case)
    N = g.num_nodes()
    if case == "tile_plus_1":
        assert N % 128 == 1
    dg = prepare_graph(g, DEV)
    gen = torch.Generator().manual_seed(N)
    k = 1.0 / D_ ** 0.5
    mk = lambda *sh: ((torch.rand(*sh, generator=gen) * 2 - 1) * k).to(DEV)
    wf, bf, bih, whh, bhh = mk(3 * D_, D_) * 1.5, mk(3 * D_), mk(3 * D_), mk(3 * D_, D_), mk(3 * D_)
    st = _stream_ptr()
    ib = L.call("ddfa_act_image_bytes", N)
    h32 = torch.tanh(torch.randn(N, D_, generator=gen)).to(DEV)
    h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_act_to_image", _p(h32), N, D_, _p(h_img), st)
    s_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gather_sum_image_src", _p(dg.indptr), _p(dg.indices), _p(h_img), N, D_, _p(s_img), st)
    wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D_, ENGINE_TCGEN05)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare", _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), D_, ENGINE_TCGEN05, _p(ws), wsb, st)
    gates = torch.empty(L.call("ddfa_gru_gates_packed_bytes", N, D_), dtype=torch.uint8, device=DEV)
    o_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D_, None, _p(o_img), _p(gates), _p(ws), wsb, st)

    wsb_b = L.call("ddfa_gru_step_bwd_workspace_bytes", N, D_, ENGINE_TCGEN05)
    ws_b = torch.empty(wsb_b, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare_bwd", _p(wf), _p(whh), D_, ENGINE_TCGEN05, _p(ws_b), wsb_b, st)
    dpart = torch.randn(N, D_, generator=gen).to(DEV)
    ds_prev = torch.randn(N, D_, generator=gen).to(DEV)
    shapes = dict(dwf=(3 * D_, D_), dbf=(3 * D_,), dbih=(3 * D_,), dwhh=(3 * D_, D_), dbhh=(3 * D_,))
    default = L.call("ddfa_tuning_get", TUNE_GATE_BWD_TMA)
    outs = {}
    try:
        for mode in (2, 1, 0):
            L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, mode)
            for step0 in (False, True):            # step 0 hands h over as fp32 rows (h_0 = x), later steps as the image
                got = dict(ds=torch.full((N, D_), float("nan"), device=DEV), dh=torch.full((N, D_), float("nan"), device=DEV))
                got.update({n: torch.zeros(shapes[n], device=DEV) for n in GRADS})
                L.call("ddfa_gru_step_bwd_image_v2", _p(dpart), _p(ds_prev), _p(dg.indptr_t), _p(dg.indices_t), _p(h32) if step0 else None,
                       _p(h_img), _p(s_img), _p(gates), _p(dg.indptr), N, D_, _p(got["ds"]), _p(got["dh"]), *[_p(got[n]) for n in GRADS],
                       _p(ws_b), wsb_b, 0, st)
                torch.cuda.synchronize()
                outs[(mode, step0)] = got
    finally:
        L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, default)
    for (mode, step0), a in outs.items():
        if mode == 0:
            continue
        b = outs[(0, step0)]
        assert not torch.isnan(a["ds"]).any() and not torch.isnan(a["dh"]).any(), (case, mode, step0)
        for n in ("ds", "dh", "dwf", "dwhh"):
            assert torch.equal(a[n], b[n]), (case, mode, step0, n, float((a[n] - b[n]).abs().max()))
        for n in BIASES:
            assert float((a[n] - b[n]).abs().max()) <= 1e-4 * max(1e-30, float(b[n].abs().max())), (case, mode, step0, n)


def test_fused_bwd_rejects_dh_aliasing_ds_prev(L):
    """Phase B of one cluster writes dh while phase A of another still gathers ds_prev rows: the two must be distinct."""
    N = 256
    buf = torch.zeros(N, D_, device=DEV)
    one = torch.zeros(16, device=DEV)
    with pytest.raises(DdfaError, match="dh must not alias ds_prev"):
        L.call("ddfa_gru_step_bwd_image_v2", _p(one), _p(buf), _p(one), _p(one), None, _p(one), _p(one), _p(one), _p(one), N, D_,
               _p(one), _p(buf), *[_p(one)] * 5, _p(one), 16, 0, _stream_ptr())


def test_fused_trainer_cuda_graph_replay_matches_eager():
    """A whole FusedTrainer step with the fused backward kernel, captured in a CUDA graph: replays give the eager loss curve."""
    batches = [synth.make_batch(64, 60, seed=90 + i, vuln_rate=0.3) for i in range(2)]
    losses = {}
    for mode in ("eager", "graph"):
        torch.manual_seed(1)
        m = D.FlowGNNGGNNModule(FEAT, 1002, 32, 4, 2, concat_all_absdf=True, engine="tcgen05").to(DEV)
        tr = D.FusedTrainer(m, use_cuda_graph=(mode == "graph"))
        bs = [b.to(DEV) for b in batches]
        losses[mode] = [float(tr.step(bs[i % 2])) for i in range(6)]      # eager warm-up, capture, then replays
        if mode == "graph":
            assert len(tr._graphs) == 2
    for a, b in zip(losses["eager"], losses["graph"]):
        assert abs(a - b) < 1e-5 * max(1.0, abs(a)), losses
    assert losses["eager"][0] != losses["eager"][2]
