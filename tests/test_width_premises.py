"""CPU: the widths and shapes of tests/test_width_gpu.py still reach every dispatch path of the SIMT engine those tests are written
for — the sgemm kernels and their K splits, the gather instances, the gate-backward and embedding-backward launch shapes, the
deterministic embedding's team forms (tests/width_batches.py restates the launch formulas).  Fails if a shape is shrunk below its
purpose.  Also: the module refuses, at construction, the widths and engine choices no kernel runs."""
import pytest

import deepdfa_b200 as D
from deepdfa_b200.module import MAX_HIDDEN_WIDTH
from width_batches import (C1_NODES, DET_CHUNK, GATE_BWD_ROWS, MAX_WIDTH, NUM_SMS, SGEMM_EDGES, WIDTHS, embed_bwd_launch, embed_det_launch,
                           engine_sgemm_calls, gate_bwd_launch, gather_instance, ordered_plan, sgemm_plan, simt_wgrad_split)

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


def _plans(deterministic=False):
    out = {}
    for W in WIDTHS:
        for name, (ta, tb, M, N, K, beta, split) in engine_sgemm_calls(W, C1_NODES).items():
            out[(W, name)] = sgemm_plan(M, N, K, beta, split, deterministic)
    return out


def test_engine_calls_reach_every_sgemm_path():
    plans = _plans()
    for W in WIDTHS:
        assert plans[(W, "fwd gi/gh")]["kernel"] == "big" and plans[(W, "dgrad ds")]["kernel"] == "big"
        wg = plans[(W, "wgrad")]
        assert wg["kernel"] == "big" and wg["atomic"] and wg["z"] > 1            # the weight gradient: atomic split-K at K = N
    assert C1_NODES > 150_000
    # 3W below one 128-column tile (W = 20, 32): the weight gradient runs one mostly-empty 128x128 tile per slice
    assert {W for W in WIDTHS if 3 * W < 128} == {20, 32}
    assert any(3 * W % 128 for W in WIDTHS if 3 * W > 128)                        # a ragged last tile of 3W (W = 96: 288)
    # the fold on both kernels: small up to 3W^2 <= 512^2, the 128x128 kernel at W = 512
    assert plans[(512, "fold fwd")]["kernel"] == "big" and plans[(256, "fold fwd")]["kernel"] == "small"
    # the small kernel with and without its K split (beta == 1, K >= 256, fewer tiles than SMs)
    small = [p for p in plans.values() if p["kernel"] == "small"]
    assert any(p["z"] > 1 and p["atomic"] for p in small) and any(p["z"] == 1 for p in small)
    assert plans[(96, "fold bwd dW")]["z"] > 1 and plans[(20, "head wgrad")]["z"] > 1
    # in deterministic mode no small-kernel call splits K, and ddfa_sgemm refuses split_k > 1
    det = _plans(deterministic=True)
    assert all(p["z"] == 1 for p in det.values() if p["kernel"] == "small")
    assert all(det[(W, "wgrad")]["kernel"] == "refused" for W in WIDTHS)


def test_ordered_split_has_a_ragged_last_slice():
    """sgemm_splitk_ordered (the deterministic weight gradient) at C1: many slices, the last one shorter than the others."""
    ragged = []
    for W in WIDTHS:
        p = ordered_plan(C1_NODES, simt_wgrad_split(C1_NODES, W))
        assert p["nz"] >= 2 and 0 < p["last"] <= p["kps"]
        if p["last"] < p["kps"]:
            ragged.append(W)
    assert 20 in ragged and 512 in ragged, ragged
    assert ordered_plan(C1_NODES, simt_wgrad_split(C1_NODES, 20))["nz"] > 100      # W = 20: hundreds of slices


def test_sgemm_edges_sit_on_either_side_of_each_boundary():
    p = {k: sgemm_plan(M, N, K, beta) for k, (ta, tb, M, N, K, alpha, beta) in SGEMM_EDGES.items()}
    e = SGEMM_EDGES
    assert e["mn=512^2"][2] * e["mn=512^2"][3] == 512 * 512 and p["mn=512^2"]["kernel"] == "small"
    assert e["mn=512^2+1"][2] * e["mn=512^2+1"][3] == 512 * 512 + 1 and p["mn=512^2+1"]["kernel"] == "big"
    assert p["mn=512x513"]["kernel"] == "big"
    assert p["k=4096"]["kernel"] == "small" and p["k=4097"]["kernel"] == "big"
    assert p["k=255,beta=1"]["z"] == 1 and p["k=256,beta=1"]["z"] > 1 and p["k=256,beta=1"]["kernel"] == "small"
    assert p["tiles=131"]["tiles"] == NUM_SMS - 1 and p["tiles=131"]["z"] > 1
    assert p["tiles=132"]["tiles"] == NUM_SMS and p["tiles=132"]["z"] == 1 and p["tiles=132"]["kernel"] == "small"
    assert p["small,alpha,beta=0.5"]["kernel"] == "small" and p["big,alpha,beta=0.5"]["kernel"] == "big"
    assert all(e[k][5] != 1.0 for k in ("small,alpha,beta=0.5", "big,alpha,beta=0.5", "big,beta=1"))
    assert {b for *_, b in e.values()} == {0.0, 0.5, 1.0}
    # deterministic mode: the beta == 1, K >= 256 small shapes run without the RED.ADD split
    assert sgemm_plan(64, 64, 256, 1.0, deterministic=True)["z"] == 1


def test_every_reachable_gather_instance_is_covered():
    covered = {gather_instance(W) for W in WIDTHS if W != 128}
    assert covered == {(8, 1), (16, 1), (32, 1), (32, 2), (32, 4)}
    assert gather_instance(20) == (8, 1) and 20 // 4 < 8                        # three idle lanes per group
    assert gather_instance(96) == (32, 1)
    assert gather_instance(1024) == (32, 8) and max(WIDTHS) < 1024               # the CH = 8 instance is past the module's limit


def test_launch_shapes_of_the_gate_and_embedding_backward():
    gb = gate_bwd_launch(C1_NODES, 20)
    assert gb["block"] == (5, 51) and gb["rows_per_thread"] == 3 and gb["ctas"] > 1000
    assert GATE_BWD_ROWS % gb["block"][1]                                         # 51 rows per pass: a ragged last pass per CTA
    for W in WIDTHS:
        g = gate_bwd_launch(C1_NODES, W)
        assert g["block"][0] * g["block"][1] <= 256 and g["smem"] <= 48 * 1024
    assert gate_bwd_launch(C1_NODES, 512)["block"] == (128, 2)
    assert C1_NODES % GATE_BWD_ROWS                                               # a ragged last gate-backward CTA
    # default embedding backward: blockDim.y >= 2 (the two hot rows are summed by threadIdx.y 0 and 1)
    for W, (K, H) in WIDTHS.items():
        b = embed_bwd_launch(C1_NODES, K, H)
        assert b["block"][1] >= 2 and b["block"][0] * b["block"][1] <= 256
    assert embed_bwd_launch(C1_NODES, 1, 512)["block"] == (128, 2)
    # deterministic embedding backward: every team form the widths reach
    forms = {W: embed_det_launch(C1_NODES, H) for W, (K, H) in WIDTHS.items()}
    assert {f["COLS"] for f in forms.values()} == {1, 4} and forms[512]["COLS"] == 4
    assert forms[48]["TL"] == 4 and forms[20]["TL"] == 8                         # H / 4 = 3 and 5: teams wider than the row
    assert forms[512]["TL"] == 32 and 512 // 4 == forms[512]["TL"] * forms[512]["COLS"]
    assert forms[20]["chunks"] > 600 and C1_NODES % DET_CHUNK                   # index 0 spans hundreds of chunks


# ---- the module refuses, at construction, what no kernel runs -------------------------------------------------------------
def test_constructor_rejects_widths_past_the_kernels():
    assert max(WIDTHS) == MAX_WIDTH == MAX_HIDDEN_WIDTH                          # the GPU tests run the widest width accepted
    with pytest.raises(ValueError, match=r"640.*hidden_dim=160, concat_all_absdf=True.*512"):
        D.FlowGNNGGNNModule(FEAT, 50, 160, 2, 1, concat_all_absdf=True)
    with pytest.raises(ValueError, match=r"516.*hidden_dim=516, concat_all_absdf=False.*512"):
        D.FlowGNNGGNNModule(FEAT, 50, 516, 2, 1, engine="simt")
    m = D.FlowGNNGGNNModule(FEAT, 50, 512, 2, 1)                                  # the widest the kernels run builds
    assert m.engine == "simt" and m._D == 512
    m4 = D.FlowGNNGGNNModule(FEAT, 50, 128, 2, 1, concat_all_absdf=True)          # W = 512 as four tables
    assert m4._D == 512


def test_constructor_rejects_tcgen05_at_other_widths(monkeypatch):
    monkeypatch.delenv("DDFA_B200_ENGINE", raising=False)
    with pytest.raises(ValueError, match=r"tcgen05.*engine argument.*128.*64 \(hidden_dim=16, concat_all_absdf=True\)"):
        D.FlowGNNGGNNModule(FEAT, 50, 16, 2, 1, concat_all_absdf=True, engine="tcgen05")
    monkeypatch.setenv("DDFA_B200_ENGINE", "tcgen05")
    with pytest.raises(ValueError, match=r"DDFA_B200_ENGINE.*128.*32 \(hidden_dim=32, concat_all_absdf=False\)"):
        D.FlowGNNGGNNModule(FEAT, 50, 32, 2, 1)
    assert D.FlowGNNGGNNModule(FEAT, 50, 32, 2, 1, concat_all_absdf=True).engine == "tcgen05"     # W = 128
    assert D.FlowGNNGGNNModule(FEAT, 50, 32, 2, 1, engine="simt").engine == "simt"                # the argument wins
    monkeypatch.delenv("DDFA_B200_ENGINE")
    assert D.FlowGNNGGNNModule(FEAT, 50, 128, 2, 1).engine == "tcgen05"                           # default at W = 128
    assert D.FlowGNNGGNNModule(FEAT, 50, 24, 2, 1, concat_all_absdf=True).engine == "simt"        # W = 96
