"""GPU: the fused backward GRU step's ds / dh tensor-map copies when the last tile ends at or just past warpgroup 1's first row.

Each warpgroup of bwd_step_fused_kernel writes its 64 rows of a tile as [64 x 32] boxes, which the tensor maps clip at row N.
N = 128 k + 64 leaves warpgroup 1 of the last tile no row (it issues nothing) and N = 128 k + 65 leaves it one row of a box.
As in test_bwd_epilogue_gpu.py: rows past N stay untouched and every row below N is bit-equal to the two-kernel path."""
import pytest
import torch

from deepdfa_b200 import synth
from deepdfa_b200._lib import TUNE_GATE_BWD_TMA, lib
from test_bwd_epilogue_gpu import _bits_equal, _Step, _untouched

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tail", [64, 65])
def test_fused_epilogue_last_box_partial_or_empty(tail):
    L = lib()
    g = synth.make_batch(seed=36 + tail, sizes=[125] * 40 + [120 + tail])      # 128 x 40 + tail nodes
    assert g.num_nodes() % 128 == tail
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
        assert _untouched(bs, N) and _untouched(bh, N), (tail, mode, step0, "a row past N was written")
        if mode == 0:
            continue
        rs, rh = got[(0, step0)]
        assert not torch.isnan(bs[:N]).any() and not torch.isnan(bh[:N]).any(), (tail, mode, step0)
        assert _bits_equal(bs[:N], rs[:N]), (tail, mode, step0, "ds", float((bs[:N] - rs[:N]).abs().max()))
        assert _bits_equal(bh[:N], rh[:N]), (tail, mode, step0, "dh", float((bh[:N] - rh[:N]).abs().max()))
