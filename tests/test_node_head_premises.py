"""CPU: the cases of tests/test_node_head_width_gpu.py and tests/test_statement_kernels_gpu.py still reach the tails of the launch
shapes they are written for (head_batches.py and statement_rule.py restate them): a K that is not a multiple of the GEMM's k step,
row counts that are not a multiple of the 64-row tile, empty weight-gradient chunks, node counts that are not a multiple of the
8 rows of a warp-per-row CTA, more functions than the shap and metric grids have CTAs, functions longer than one metric CTA.
Also: the float64 chain of head_batches.node_head_ref is torch.autograd's, and its bounds hold for an fp32 evaluation."""
import numpy as np
import pytest
import torch

import head_batches as H
import statement_rule as R
from scale_batches import HUB_SHAPES
from width_batches import C1_NODES

HUB_NODES = HUB_SHAPES["mid"][2]


def test_widths_reach_the_ragged_k_step_and_the_wide_shapes():
    Ks = [2 * D for D in H.NODE_HEAD_WIDTHS]
    assert any(K % H.NODE_HEAD_BK for K in Ks)                       # D = 20: K = 40, a half k step at the end
    assert max(Ks) == 1024 and any(K % 64 for K in Ks)               # the widest head; a ragged last 64-column tile
    assert {192, 256, 320, 384, 448, 512} <= set(H.NODE_HEAD_WIDTHS)   # every width of the tensor-core wide engine
    # the largest C1 case needs a workspace above 1.3 GB, and with the planes and the float64 reference stays far below 80 GB
    ws = H.node_head_ws_bytes(C1_NODES, 512)
    assert 1.3e9 < ws < 2e9


def test_c1_row_list_is_like_the_trainers_and_ragged():
    rows = H.node_rows_trainer(C1_NODES, seed=512)
    S = len(rows)
    assert rows[0] == 0 and rows[-1] == C1_NODES - 1 and np.all(np.diff(rows) > 0)
    assert 0.2 * C1_NODES < S < 0.4 * C1_NODES and S % H.NODE_HEAD_BM != 0
    for D in H.NODE_HEAD_WIDTHS:
        r = H.node_rows_trainer(C1_NODES, seed=D + 1)      # the seeds of test_head_at_c1_every_width
        assert len(r) % H.NODE_HEAD_BM, D
    chunks = H.node_head_chunks(C1_NODES)                            # every row: chunks of 4 919 rows, the last one shorter
    assert chunks[0] == (0, 4919) and chunks[-1][1] == C1_NODES and chunks[-1][1] - chunks[-1][0] < 4919


def test_small_row_counts_leave_chunks_empty():
    empty = {}
    for S in H.NODE_SMALL_S:
        S = HUB_NODES if S < 0 else S
        ch = H.node_head_chunks(S)
        assert sum(r1 - r0 for r0, r1 in ch) == S and all(ch[i][1] == ch[i + 1][0] for i in range(len(ch) - 1))
        empty[S] = sum(r1 == r0 for r0, r1 in ch)
    assert empty[0] == 32 and empty[1] == 31 and empty[5] == 27 and empty[31] == 1 and empty[32] == 0
    assert empty[33] == 15                                          # chunks of 2 rows: the 17th holds one, 15 are empty
    rows = H.node_rows(HUB_NODES, 5, 1)
    assert HUB_NODES - 1 in rows and 0 in rows and len(set(rows.tolist())) == 5
    assert list(H.node_rows(HUB_NODES, 1, 0)) == [HUB_NODES - 1]


def test_warp_per_row_kernels_get_a_ragged_last_cta():
    for N in (C1_NODES, HUB_NODES, 613):                            # head_out_kernel, input_grad_score_kernel, node_probability
        assert N % H.NODE_HEAD_WARP_ROWS and N % R.SCORE_WARP_ROWS, N
    assert any(D % 32 for D in R.SCORE_WIDTHS) and any(D < 32 for D in R.SCORE_WIDTHS) and max(R.SCORE_WIDTHS) == 512


def test_shap_and_metric_cases_stride_over_their_grids():
    sizes = R.shap_sizes(0)
    assert len(sizes) > R.SHAP_MAX_CTAS and (sizes == 0).any() and sizes[-1] == 0
    assert R.SHAP_COUNTER >= 2 ** 32 and all(D % 4 == 0 for D in R.SHAP_WIDTHS)
    s, v, bnn = R.metric_case()
    assert len(bnn) > R.STMT_MAX_CTAS and bnn.max() == 20_000 and (bnn > R.STMT_THREADS).sum() >= 5
    ranks = R.ranks(s, v, bnn)
    assert sum(r[3] for r in ranks[:580]) == 1                    # one NaN function among the valid ones
    # the 20 000-node function: the first-ranked vulnerable node is node 97 (warp 3, first iteration), tied at the top with
    # vulnerable nodes of lower warps and later iterations
    assert ranks[0][1] == 2
    tied = np.nonzero((v[:20_000] != 0) & (s[:20_000] == s[:20_000].max()))[0]
    assert tied.min() == 97 and len({(n % R.STMT_THREADS) // 32 for n in tied}) >= 2 and len({n // R.STMT_THREADS for n in tied}) >= 3
    # the 1 000-node function: its first-ranked vulnerable node is in the last warp of a late iteration
    n0 = 20_000
    sv = np.where(v[n0:n0 + 1000] != 0, s[n0:n0 + 1000], -np.inf)
    best = int(np.argmax(sv))
    assert (best % R.STMT_THREADS) // 32 == 3 and best // R.STMT_THREADS == 3 and ranks[1][1] == 3
    # signed zeros: -0.0 ranks with the +0.0 nodes before it; a lower vulnerable +0.0 ranks first
    assert ranks[2][1] == 2 and ranks[3][1] == 1


def test_node_head_ref_is_autograd_and_its_bounds_hold():
    """On a small case in float32 on the CPU: node_head_ref's float64 chain equals torch.autograd of the head with each hidden ReLU
    masked by the float32 forward's side and each stage fed the float32 forward's values, and the float32 forward / backward is inside every bound."""
    torch.manual_seed(0)
    S, D, L = 200, 20, 3
    ws, bs = H.mlp_params(D, L, 3)
    ins0 = torch.randn(S, 2 * D)
    dl = torch.randn(S)
    dw0 = [torch.randn(w.shape) for w in ws]
    db0 = [torch.randn(b.shape) for b in bs]
    acts, a = [], ins0
    for i in range(L - 1):
        a = torch.relu(a @ ws[i].t() + bs[i])
        acts.append(a)
    ref = H.node_head_ref(ins0, acts, ws, bs, dl, dw0, db0)
    # autograd, float64, relu(z) read as z * mask of the float32 forward, each hidden value the float32 forward's (the gradient
    # of z * mask, the value of act)
    o = ins0.double().requires_grad_(True)
    w64 = [w.double().requires_grad_(True) for w in ws]
    b64 = [b.double().requires_grad_(True) for b in bs]
    z = o
    for i in range(L):
        z = z @ w64[i].t() + b64[i]
        if i < L - 1:
            zm = z * (acts[i] > 0).double()
            z = acts[i].double() + (zm - zm.detach())
    z.reshape(-1).backward(dl.double())
    torch.testing.assert_close(ref["din"][0], o.grad, rtol=1e-12, atol=1e-12)
    for i in range(L):
        torch.testing.assert_close(ref[f"dw{i}"][0], w64[i].grad + dw0[i].double(), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(ref[f"db{i}"][0], b64[i].grad + db0[i].double(), rtol=1e-12, atol=1e-12)
    # the float32 evaluation of the same chain is within the bounds
    g = dl[:, None]
    got = {}
    for i in range(L - 1, -1, -1):
        got[f"dw{i}"] = dw0[i] + g.t() @ (acts[i - 1] if i else ins0)
        got[f"db{i}"] = db0[i] + g.sum(0)
        g = g @ ws[i]
        if i:
            g = g * (acts[i - 1] > 0)
    got["din"] = g
    for k, v in got.items():
        r, mag, tau = ref[k]
        assert H.ratio((v.double() - r).abs(), tau * mag) <= 1.0, k
