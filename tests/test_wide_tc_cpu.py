"""CPU: which widths the tensor-core engine accepts (argument and DDFA_B200_ENGINE), the unchanged default engine, and the launch
shapes of the wide-width GEMMs (tests/wide_tc_shapes.py restates csrc/gru_tc_wide.cu): the widths and node count of
tests/test_wide_tc_gpu.py must reach every tail case of the kernel."""
import pytest

import deepdfa_b200 as D
from deepdfa_b200._lib import ENGINE_SIMT, ENGINE_TCGEN05, lib
from deepdfa_b200.module import MAX_HIDDEN_WIDTH, TCGEN05_WIDTHS, default_engine
from wide_tc_shapes import WIDE_WIDTHS, gemm_launches, wgrad_slices
from width_batches import C1_NODES

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
ACCEPTED = {128, *WIDE_WIDTHS}


def _module(W, **kw):
    """A module of hidden width W: concat_all_absdf with hidden_dim W / 4 where W % 16 == 0, else one table of W columns."""
    if W % 16 == 0:
        return D.FlowGNNGGNNModule(FEAT, 50, W // 4, 2, 1, concat_all_absdf=True, **kw)
    return D.FlowGNNGGNNModule(FEAT, 50, W, 2, 1, **kw)


def test_accepted_widths():
    assert set(TCGEN05_WIDTHS) == ACCEPTED
    assert WIDE_WIDTHS == tuple(range(192, MAX_HIDDEN_WIDTH + 1, 64))


@pytest.mark.parametrize("source", ["argument", "environment"])
def test_constructor_accepts_and_refuses_tcgen05(source, monkeypatch):
    monkeypatch.delenv("DDFA_B200_ENGINE", raising=False)
    kw = {"engine": "tcgen05"}
    if source == "environment":
        monkeypatch.setenv("DDFA_B200_ENGINE", "tcgen05")
        kw = {}
    for W in range(4, MAX_HIDDEN_WIDTH + 1, 4):
        if W in ACCEPTED:
            m = _module(W, **kw)
            assert m.engine == "tcgen05" and m._D == W
        else:
            where = "engine argument" if source == "argument" else "DDFA_B200_ENGINE"
            with pytest.raises(ValueError, match=rf"tcgen05.*{where}.*128, 192, 256, 320, 384, 448 and 512 only, got {W} \(hidden_dim="):
                _module(W, **kw)


def test_default_engine_is_unchanged(monkeypatch):
    monkeypatch.delenv("DDFA_B200_ENGINE", raising=False)
    for W in range(4, MAX_HIDDEN_WIDTH + 1, 4):
        want = "tcgen05" if W == 128 else "simt"
        assert default_engine(W) == want
        assert _module(W).engine == want


def test_step_workspaces_and_refusals():
    L = lib()
    for W in range(64, MAX_HIDDEN_WIDTH + 1, 32):
        fwd = L.call("ddfa_gru_step_workspace_bytes", C1_NODES, W, ENGINE_TCGEN05)
        bwd = L.call("ddfa_gru_step_bwd_workspace_bytes", C1_NODES, W, ENGINE_TCGEN05)
        ggnn = L.call("ddfa_ggnn_workspace_bytes", C1_NODES, W, 8, ENGINE_TCGEN05, 1)
        if W in WIDE_WIDTHS:
            # at least the SIMT layout: the wide path keeps its planes and adds the operand images
            assert fwd > L.call("ddfa_gru_step_workspace_bytes", C1_NODES, W, ENGINE_SIMT)
            assert bwd > L.call("ddfa_gru_step_bwd_workspace_bytes", C1_NODES, W, ENGINE_SIMT)
            assert ggnn > 0
            assert L.call("ddfa_gru_tc_wide_gemm_workspace_bytes", 3, C1_NODES, W) > 0
        elif W != 128:
            assert fwd == 16 and bwd == 16 and ggnn == 0
            assert L.call("ddfa_gru_tc_wide_gemm_workspace_bytes", 0, C1_NODES, W) == 0


@pytest.mark.parametrize("W", WIDE_WIDTHS)
@pytest.mark.parametrize("N", [1, 63, 64, 65, 127, 129, 1000, C1_NODES])
def test_wgrad_slices_match_the_library(W, N):
    sl = wgrad_slices(N, W)
    assert L_slices(N, W) == sl["nz"]
    assert 1 <= sl["nz"] <= 32 and 1 <= sl["last"] <= sl["kps"]
    assert (sl["nz"] - 1) * sl["kps"] < sl["nks"] <= sl["nz"] * sl["kps"]      # every slice has work, none is left out


def L_slices(N, W):
    return lib().call("ddfa_gru_tc_wide_wgrad_slices", N, W)


def test_gpu_shapes_reach_every_tail_case():
    """At N = 157 381 over the widths of the GPU test: node tiles ragged to 128 and to 64; 128-wide column tiles both full and with
    one valid half, in the M (weight gradient) and the N (forward, dgrad) position; odd and even K step counts; a weight gradient
    whose last slice is shorter than the others and one whose slices are all equal; and the one-wave fill of the split."""
    assert C1_NODES % 128 not in (0, 64) and C1_NODES % 64 != 0
    seen = set()
    for W in WIDE_WIDTHS:
        sh = gemm_launches(C1_NODES, W)
        assert sh["fwd"]["m_ragged"] == C1_NODES % 128
        for name in ("fwd", "dgrad"):
            seen.add((name, "n_half", sh[name]["n_half"]))
            seen.add((name, "odd_k", sh[name]["nks"] % 2 == 1))
        seen.add(("wgrad", "m_half", sh["wgrad"]["m_half"]))
        seen.add(("wgrad", "n_half", sh["wgrad"]["n_half"]))
        sl = wgrad_slices(C1_NODES, W)
        seen.add(("wgrad", "ragged_last", sl["last"] < sl["kps"]))
        assert sh["wgrad"]["ctas"] <= 32 * 132
    for case in [("fwd", "n_half"), ("dgrad", "n_half"), ("wgrad", "m_half"), ("wgrad", "n_half"), ("fwd", "odd_k"), ("dgrad", "odd_k"),
                 ("wgrad", "ragged_last")]:
        assert (*case, True) in seen and (*case, False) in seen, case
    # W = 256 and W = 512 fill whole waves of the 132 SMs: 12 tiles x 11 slices and 48 tiles x 11 slices
    assert gemm_launches(C1_NODES, 256)["wgrad"]["ctas"] == 132
    assert gemm_launches(C1_NODES, 512)["wgrad"]["ctas"] == 528
