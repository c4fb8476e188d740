"""CPU: the host references of tests/test_head_gpu.py are right, and its shapes still reach the edges those tests are written for
— the Philox known answers, the sampler's tie at the threshold key across two CTAs, the batched-MLP switch, ragged row slices of
the bias-gradient sum, graphs of 0, 1 and 40 000 nodes.  Fails if a shape is changed below its purpose."""
import numpy as np
import pytest
import torch

import head_batches as H
from deepdfa_b200.engine import undersample_count


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_host_philox_reproduces_random123_known_answers(ctr, key, want):
    assert tuple(int(w) for w in H.philox4x32_10(ctr, key)) == want


def test_node_keys_put_the_draw_in_the_counter():
    k = H.node_keys(8, (5 << 32) + 9, (3 << 32) + 7)
    for n in range(8):
        assert int(k[n]) == int(H.philox4x32_10((7, 3, n, 0), (9, 5))[0])


def test_sample_ref_takes_the_smallest_keys_ties_in_node_order():
    vuln = np.array([0, 1, 0, 0, 0, 0], np.int32)
    keys = H.node_keys(6, 0, 0)
    rows, S, over, nxt = H.sample_ref(vuln, 6, 2.0, 0, 0)
    pop = [0, 2, 3, 4, 5]
    take = sorted(sorted(pop, key=lambda n: (int(keys[n]), n))[:2])
    assert list(rows) == sorted([1] + take) and S == 3 and not over and nxt == 1
    rows, S, over, _ = H.sample_ref(vuln, 4, 10.0, 0, 0)          # k = 10 > 3: the whole valid population, overflow
    assert list(rows) == [0, 1, 2, 3] and over
    rows, S, over, nxt = H.sample_ref(vuln, 4, -1.0, 0, 7)        # no undersampling: no draw
    assert list(rows) == [0, 1, 2, 3] and nxt == 7


def test_tie_case_exists_across_sampler_ctas():
    t = H.tie_case()
    assert t is not None
    v = t["vuln"]
    assert len(v) == H.c1_batch().num_nodes() > 150_000
    a, b = t["a"], t["b"]
    keys = H.node_keys(len(v), t["seed"], 0)
    assert a < b and a // H.SAMPLER_CTA_NODES != b // H.SAMPLER_CTA_NODES
    assert keys[a] == keys[b] == t["key"] and int(np.count_nonzero(keys == t["key"])) == 2
    assert v[a] == 0 and v[b] == 0 and t["n_vuln"] > 0
    assert t["k_a"] == t["below"] + 1 and t["k_ab"] == t["below"] + 2
    ra, *_ = H.sample_ref(v, len(v), t["factor_a"], t["seed"], 0)
    rab, *_ = H.sample_ref(v, len(v), t["factor_ab"], t["seed"], 0)
    assert a in ra and b not in ra and a in rab and b in rab


def test_sampler_cases_reach_their_edges():
    cases = {c[0]: c for c in H.sampler_cases()}
    _, v, nv, f, _, _ = cases["ragged_N"]
    assert len(v) % H.SAMPLER_CTA_NODES and len(v) > 4 * H.SAMPLER_CTA_NODES
    assert cases["num_valid_0"][2] == 0 and len(cases["N1_clean"][1]) == 1
    _, v, nv, f, _, _ = cases["padding"]
    assert nv < len(v) and v[nv:].all()
    _, v, nv, f, s, d = cases["k0"]
    assert undersample_count(int(v.sum()), f) == 0
    _, v, nv, f, s, d = cases["k_pop"]
    assert undersample_count(int(v[:nv].sum()), f) == int((v[:nv] == 0).sum())
    assert H.sample_ref(*cases["k_over"][1:])[2] and H.sample_ref(*cases["N1_vuln"][1:])[2]
    assert not H.sample_ref(*cases["k_pop"][1:])[2]
    for name, want in (("half_5x0.5", 2), ("half_7x0.5", 4), ("half_3x1.5", 4)):
        _, v, nv, f, _, _ = cases[name]
        prod = int(v.sum()) * f
        assert prod % 1 == 0.5 and undersample_count(int(v.sum()), f) == want
    assert cases["draw_hi"][5] >> 32
    assert cases["c1"][2] > 150_000


def test_readout_shapes_reach_their_edges():
    c1 = H.c1_sizes()
    assert len(c1) == 1024 and c1.sum() > 150_000 and len(c1) >= H.BATCHED_MLP_MIN_B
    big = H.big_sizes()
    assert H.HUGE_GRAPH in big and big.sum() > H.HUGE_GRAPH and len(big) < H.BATCHED_MLP_MIN_B
    mid = len(big) // 2
    for part in (big[:3], big[mid - 10:mid + 10], big[-3:]):
        assert 0 in part and 1 in part
    mixed = H.mixed_sizes()
    assert len(mixed) < H.BATCHED_MLP_MIN_B and 0 in mixed and 1 in mixed and mixed.max() > 512
    sw = H.switch_sizes()
    assert len(sw) == H.BATCHED_MLP_MIN_B and sw.min() >= 1


def test_mlp_bwd_batches_take_ragged_row_slices():
    assert H.colsum_slices(1000) > 1 and 1000 % H.colsum_slices(1000) != 0
    assert H.colsum_slices(1024) > 1 and H.colsum_slices(255) == 1


def test_extreme_gate_logits_overflow_without_the_max():
    sizes = H.big_sizes()
    h, x, w, b = H.readout_inputs(sizes, 128, 3, extreme=True)
    g = torch.cat([h, x], 1).double() @ w.double() + float(b[0])
    assert float(g.max()) > 88.8                             # expf overflows above ~88.72
    j = int(np.argmax(sizes))
    gp = H.graph_ptr(sizes).long()
    gj = g[int(gp[j]):int(gp[j + 1])]
    assert float(gj.max() - gj.min()) > 199 and float((torch.exp((gj - gj.max()).float()) == 0).double().mean()) > 0.3


def test_readout_bwd_ref_is_the_autograd_gradient():
    """The explicit chain rule of readout_bwd_ref against fp64 autograd of the attention pooling (exact saved state)."""
    sizes = np.array([3, 0, 1, 7])
    D = 4
    h, x, w, b = H.readout_inputs(sizes, D, 1)
    o = torch.cat([h, x], 1).double().requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    b64 = b.double().requires_grad_(True)
    seg = H.segment_ids(sizes)
    g = o @ w64 + b64
    B = len(sizes)
    M = torch.full((B,), -np.inf, dtype=torch.float64).scatter_reduce(0, seg, g.detach(), "amax")
    e = torch.exp(g - M[seg])
    S = torch.zeros(B, dtype=torch.float64).index_add(0, seg, e)
    pooled = torch.zeros(B, 2 * D, dtype=torch.float64).index_add(0, seg, (e / S[seg])[:, None] * o)
    dp = torch.randn(B, 2 * D, dtype=torch.float64)
    (pooled * dp).sum().backward()
    r = H.readout_bwd_ref(h.double(), x.double(), w.double(), sizes, dp, pooled.detach(), g.detach(), M, S.detach(),
                          torch.zeros(2 * D, dtype=torch.float64), torch.zeros(1, dtype=torch.float64))
    torch.testing.assert_close(torch.cat([r["dh"], r["dx"]], 1), o.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["dw"], w64.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["db"].reshape(1), b64.grad, rtol=1e-12, atol=1e-12)


def test_mlp_bwd_ref_is_the_autograd_gradient():
    D, L, B = 4, 3, 6
    ws, bs = H.mlp_params(D, L, 0)
    pooled = torch.randn(B, 2 * D, dtype=torch.float64, requires_grad=True)
    Wr = [w.double().requires_grad_(True) for w in ws]
    br = [b.double().requires_grad_(True) for b in bs]
    cur, acts = pooled, []
    for i in range(L):
        cur = cur @ Wr[i].t() + br[i]
        if i < L - 1:
            cur = torch.relu(cur)
            acts.append(cur.detach())
    dl = torch.randn(B, dtype=torch.float64)
    (cur.squeeze(1) * dl).sum().backward()
    z = [torch.zeros_like(w) for w in Wr]
    zb = [torch.zeros_like(b) for b in br]
    r = H.mlp_bwd_ref(dl, pooled.detach(), acts, [w.detach() for w in Wr], z, zb)
    for i in range(L):
        torch.testing.assert_close(r[i][0], Wr[i].grad, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(r[i][2], br[i].grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["dpooled"][0], pooled.grad, rtol=1e-12, atol=1e-12)
