"""GPU: the epilogue of the fused backward GRU step (bwd_step_fused_kernel), which writes ds with bulk copies and adds the
accumulator onto dh' * z in dh's rows with bulk fp32 add-reductions, both from the stage that held the last q tile.

ds and dh are unpadded [N, 128] planes: here they are views into buffers with sentinel rows (a NaN bit pattern) after row N,
which must come back untouched, while every row below N must be bit-equal to the two-kernel path (DDFA_TUNE_GATE_BWD_TMA = 0),
for h as fp32 rows (step 0) and as the image, with the folded gather's CSR data pipelined across tiles (2) and not (1).  The
CUDA-graph case chains two steps, the second reading the first one's ds and dh (the next kernel of the programmatic-launch
chain), then a plain kernel reading the second step's outputs: the bulk writes must be complete before either runs."""
import pytest
import torch

from deepdfa_b200 import synth
from deepdfa_b200._lib import ENGINE_TCGEN05, TUNE_GATE_BWD_TMA, lib
from deepdfa_b200.engine import _p, prepare_graph

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D_ = 128
KEEP0 = 16                    # DDFA_WGRAD_KEEP(0): no weight-gradient launch inside the call
SENTINEL = 0x7FC0DEAD         # a quiet-NaN bit pattern no computation produces
EXTRA = 40                    # sentinel rows after row N


def _batch(case):
    if case == "n_lt_128":
        return synth.make_batch(1, 90, seed=31)                          # one ragged tile, warpgroup 1 owns no row
    if case == "tile_plus_1":
        return synth.make_batch(seed=32, sizes=[125] * 40 + [121])       # 128 k + 1 nodes: a last tile of one row
    if case == "few_tiles":
        return synth.make_batch(9, 150, seed=33)                         # 11 tiles: fewer tiles than clusters
    return synth.make_batch(1024, 150, 2.0, 1002, seed=34)                # the benchmark's C1 batch shape


class _Step:
    """One GRU step's forward state and the backward workspace, on the current stream."""

    def __init__(self, L, g):
        self.L, self.N = L, g.num_nodes()
        N = self.N
        self.dg = dg = prepare_graph(g, DEV)
        gen = torch.Generator().manual_seed(N)
        k = 1.0 / D_ ** 0.5
        mk = lambda *sh: ((torch.rand(*sh, generator=gen) * 2 - 1) * k).to(DEV)
        wf, bf, bih, whh, bhh = mk(3 * D_, D_) * 1.5, mk(3 * D_), mk(3 * D_), mk(3 * D_, D_), mk(3 * D_)
        st = self.st = torch.cuda.current_stream().cuda_stream
        ib = L.call("ddfa_act_image_bytes", N)
        self.h32 = torch.tanh(torch.randn(N, D_, generator=gen)).to(DEV)
        self.h_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        L.call("ddfa_act_to_image", _p(self.h32), N, D_, _p(self.h_img), st)
        self.s_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gather_sum_image_src", _p(dg.indptr), _p(dg.indices), _p(self.h_img), N, D_, _p(self.s_img), st)
        wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D_, ENGINE_TCGEN05)
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare", _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), D_, ENGINE_TCGEN05, _p(ws), wsb, st)
        self.gates = torch.empty(L.call("ddfa_gru_gates_packed_bytes", N, D_), dtype=torch.uint8, device=DEV)
        o_img = torch.zeros(ib, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_fwd_image_v2", _p(self.s_img), _p(self.h_img), None, _p(dg.indptr), N, D_, None, _p(o_img), _p(self.gates),
               _p(ws), wsb, st)
        self.wsb = L.call("ddfa_gru_step_bwd_workspace_bytes", N, D_, ENGINE_TCGEN05)
        self.ws = torch.empty(self.wsb, dtype=torch.uint8, device=DEV)
        L.call("ddfa_gru_step_prepare_bwd", _p(wf), _p(whh), D_, ENGINE_TCGEN05, _p(self.ws), self.wsb, st)
        self.dpart = torch.randn(N, D_, generator=gen).to(DEV)
        self.ds_prev = torch.randn(N, D_, generator=gen).to(DEV)
        self.grads = [torch.zeros(3 * D_, D_, device=DEV), torch.zeros(3 * D_, device=DEV), torch.zeros(3 * D_, device=DEV),
                      torch.zeros(3 * D_, D_, device=DEV), torch.zeros(3 * D_, device=DEV)]

    def out(self):
        """An [N, 128] view into a buffer whose EXTRA rows after row N (and, before the call, every row) hold SENTINEL."""
        buf = torch.full((self.N + EXTRA, D_), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
        return buf, buf[:self.N]

    def bwd(self, dh_out, ds_prev, ds, dh, step0=False):
        dg = self.dg
        self.L.call("ddfa_gru_step_bwd_image_v2", _p(dh_out), _p(ds_prev), _p(dg.indptr_t), _p(dg.indices_t), _p(self.h32) if step0 else None,
                    _p(self.h_img), _p(self.s_img), _p(self.gates), _p(dg.indptr), self.N, D_, _p(ds), _p(dh), *[_p(x) for x in self.grads],
                    _p(self.ws), self.wsb, KEEP0, torch.cuda.current_stream().cuda_stream)


def _untouched(buf, N):
    return bool((buf[N:].view(torch.int32) == SENTINEL).all())


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.fixture(scope="module")
def L():
    return lib()


@pytest.mark.parametrize("case", ["n_lt_128", "tile_plus_1", "few_tiles", "c1"])
def test_fused_epilogue_rows_and_bits(L, case):
    g = _batch(case)
    if case == "tile_plus_1":
        assert g.num_nodes() % 128 == 1
    s = _Step(L, g)
    default = L.call("ddfa_tuning_get", TUNE_GATE_BWD_TMA)
    got = {}
    try:
        for mode in (0, 1, 2):
            L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, mode)
            for step0 in (False, True):
                (bs, ds), (bh, dh) = s.out(), s.out()
                s.bwd(s.dpart, s.ds_prev, ds, dh, step0)
                torch.cuda.synchronize()
                got[(mode, step0)] = (bs, bh)
    finally:
        L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, default)
    N = s.N
    for (mode, step0), (bs, bh) in got.items():
        assert _untouched(bs, N) and _untouched(bh, N), (case, mode, step0, "a row past N was written")
        if mode == 0:
            continue
        rs, rh = got[(0, step0)]
        assert not torch.isnan(bs[:N]).any() and not torch.isnan(bh[:N]).any(), (case, mode, step0)
        assert _bits_equal(bs[:N], rs[:N]), (case, mode, step0, "ds", float((bs[:N] - rs[:N]).abs().max()))
        assert _bits_equal(bh[:N], rh[:N]), (case, mode, step0, "dh", float((bh[:N] - rh[:N]).abs().max()))


def test_fused_epilogue_complete_before_successors_in_cuda_graph(L):
    """Two chained fused steps and a plain read of the second one's outputs, captured in a CUDA graph and replayed, against the
    same sequence run eagerly on the two-kernel path."""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        s = _Step(L, synth.make_batch(64, 150, seed=35))
        N = s.N
        default = L.call("ddfa_tuning_get", TUNE_GATE_BWD_TMA)
        try:
            L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, 0)
            ref = [torch.empty(N, D_, device=DEV) for _ in range(4)]
            s.bwd(s.dpart, s.ds_prev, ref[0], ref[1])
            s.bwd(ref[1], ref[0], ref[2], ref[3])
            L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, default)
            assert default != 0
            outs = [s.out() for _ in range(4)]
            ds1, dh1, ds2, dh2 = [v for _, v in outs]
            s.bwd(s.dpart, s.ds_prev, ds1, dh1)          # warm-up outside the capture (the kernel's attributes are set once)
            s.bwd(dh1, ds1, ds2, dh2)
            side.synchronize()
            for _, v in outs:
                v.view(torch.int32).fill_(SENTINEL)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                s.bwd(s.dpart, s.ds_prev, ds1, dh1)
                s.bwd(dh1, ds1, ds2, dh2)
                read = torch.cat([ds2, dh2], dim=1).clone()
            for _ in range(3):
                graph.replay()
            side.synchronize()
        finally:
            L.call("ddfa_tuning_set", TUNE_GATE_BWD_TMA, default)
    for (buf, v), r, name in zip(outs, ref, ("ds1", "dh1", "ds2", "dh2")):
        assert _untouched(buf, N), name
        assert _bits_equal(v, r), (name, float((v - r).abs().max()))
    assert _bits_equal(read, torch.cat([ref[2], ref[3]], dim=1))
