"""Shapes and host references of the head kernels — the readout (csrc/readout.cu), the MLP head and its backward, the graph loss
(csrc/loss_adam.cu) and the node-row sampler (csrc/node_loss.cu) — shared by tests/test_head_gpu.py (which runs the kernels) and
tests/test_head_premises.py (which checks on the CPU that the shapes still reach the edges the GPU tests are written for, and
that the host references are right).

Error bounds are per element and a priori: built in fp64 from the kernel's own inputs to the stage being checked, with
u = 2^-24 the unit roundoff of fp32.  A bound of the form c * K * u * (|A| |B|) is the classical bound of a length-K fp32 dot
product (any summation order), and every bound here keeps c <= 4."""
import functools

import numpy as np
import torch

from deepdfa_b200 import synth
from deepdfa_b200.engine import undersample_count
from scale_batches import MODULE_C1

U = 2.0 ** -24
ETA = 2.0 ** -150             # absolute rounding error of a result in fp32's subnormal range (half the subnormal spacing)

# ---- launch constants the tests are written against --------------------------------------------------------------------------
SAMPLER_CTA_NODES = 1024      # node_loss.cu kPerBlock: nodes per CTA of the sampler's count / write kernels
READOUT_WARPS = 8             # readout.cu kReadoutWarps: node rows of a graph are split over 8 warps
MAX_MLP_LAYERS = 16           # readout.cu kMaxMlpLayers
BATCHED_MLP_MIN_B = 256       # ddfa_readout_mlp_fwd: the batched MLP from this many graphs on (with mlp_act given)


def colsum_slices(B: int) -> int:
    """Row slices of the bias-gradient column sum in ddfa_mlp_bwd's default mode (gridDim.y of colsum_accum_kernel)."""
    return (B + 63) // 64 if B >= 256 else 1


# ---- graph-size lists of the readout / loss batches ---------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def c1_batch():
    """The benchmark's C1 batch: 1024 variable-size graphs, 157 377 nodes (also test_scale_gpu.py's module-gradient batch)."""
    return synth.make_batch(**MODULE_C1)


def c1_sizes() -> np.ndarray:
    return c1_batch().batch_num_nodes().numpy().astype(np.int64)


HUGE_GRAPH = 40_000


def big_sizes() -> np.ndarray:
    """One 40 000-node graph between ragged small ones, with empty and 1-node graphs at the start, in the middle and at the end."""
    rng = np.random.default_rng(40_000)
    a, b = rng.integers(2, 300, 40), rng.integers(2, 300, 40)
    return np.concatenate([[0, 1], a, [0, 1, HUGE_GRAPH, 1, 0], b, [1, 0]]).astype(np.int64)


def mixed_sizes(B: int = 200, seed: int = 5) -> np.ndarray:
    """B graphs of 0-700 nodes (in-CTA MLP below 256 graphs); every 37th graph is empty, every 41st has one node."""
    rng = np.random.default_rng(seed)
    s = rng.integers(2, 700, B)
    s[::37], s[5::41] = 0, 1
    return s.astype(np.int64)


def switch_sizes() -> np.ndarray:
    """256 graphs of 1-300 nodes: the first 255 are the batch below the batched-MLP switch, all 256 the batch at it."""
    return np.random.default_rng(256).integers(1, 300, 256).astype(np.int64)


# name -> (sizes, what the GPU tests rely on)
READOUT_SHAPES = {
    "c1": c1_sizes,          # training size, batched MLP
    "big": big_sizes,        # 40 000 rows in one CTA, empty / 1-node graphs at both ends and in the middle
    "mixed": mixed_sizes,    # in-CTA MLP, empty and 1-node graphs spread out
}


def graph_ptr(sizes) -> torch.Tensor:
    return torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32))


def segment_ids(sizes) -> torch.Tensor:
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.from_numpy(np.asarray(sizes, dtype=np.int64)))


# ---- readout inputs ---------------------------------------------------------------------------------------------------------
def readout_inputs(sizes, D: int, seed: int, extreme: bool = False):
    """h, x ([N, D] fp32), w_gate ([2D]), b_gate ([1]).  extreme=True: b_gate = +85 and w_gate scaled so that o.w spans +-10
    over the batch (a softmax without the running max would take exp of ~95: inf in fp32), and the rows of the largest graph
    scaled so that its logits span 200 (on the 40 000-node graph a third of its alpha underflow to 0 in fp32)."""
    gen = torch.Generator().manual_seed(seed)
    N = int(np.sum(sizes))
    h, x = torch.randn(N, D, generator=gen), torch.randn(N, D, generator=gen)
    w = torch.randn(2 * D, generator=gen) / (2 * D) ** 0.5
    b = torch.randn(1, generator=gen)
    if extreme:
        o = torch.cat([h, x], 1).double()
        w = (w.double() * (10.0 / float((o @ w.double()).abs().max()))).float()
        b = torch.tensor([85.0])
        gp = graph_ptr(sizes).long()
        j = int(np.argmax(sizes))
        n0, n1 = int(gp[j]), int(gp[j + 1])
        s = o[n0:n1] @ w.double()
        scale = 200.0 / float(s.max() - s.min())
        h[n0:n1] *= scale
        x[n0:n1] *= scale
    return h, x, w, b


def mlp_params(D: int, L: int, seed: int):
    """L linears [2D, 2D] ... [1, 2D] (He-scaled, so the activations of a deep head neither die nor blow up) and their biases."""
    gen = torch.Generator().manual_seed(1000 + seed)
    D2 = 2 * D
    ws = [torch.randn(1 if i == L - 1 else D2, D2, generator=gen) * (2.0 / D2) ** 0.5 for i in range(L)]
    bs = [0.1 * torch.randn(1 if i == L - 1 else D2, generator=gen) for i in range(L)]
    return ws, bs


# ---- readout references -----------------------------------------------------------------------------------------------------
def pool_ref(h, x, w, b, sizes):
    """fp64 gate logits, their bound, attention pooling and its first-order bound (DESIGN §4):
    |pooled_bj - ref| <= 2u [ (n_b + 2D + 8) sum_n alpha_n |o_nj| + sum_n alpha_n |o_nj - pooled_bj| (2D G_n + |g_n|) ],
    G_n = sum_k |o_nk w_k| + |b_gate|.  The first term is the accumulation (n_b online-softmax steps, the 8-warp merge, the
    division by the sum); the second is the error of each logit carried through alpha_n to the pooled vector."""
    seg = segment_ids(sizes)
    B = len(sizes)
    o = torch.cat([h, x], 1).double()
    w64, b64 = w.double(), float(b[0])
    D2 = o.shape[1]
    g = o @ w64 + b64
    G = o.abs() @ w64.abs() + abs(b64)
    M = torch.full((B,), -np.inf, dtype=torch.float64).scatter_reduce(0, seg, g, "amax")
    e = torch.exp(g - M[seg])
    S = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, e)
    a = e / S[seg]
    pooled = torch.zeros(B, D2, dtype=torch.float64).index_add_(0, seg, a[:, None] * o)
    mag = torch.zeros(B, D2, dtype=torch.float64).index_add_(0, seg, a[:, None] * o.abs())
    spread = torch.zeros(B, D2, dtype=torch.float64).index_add_(0, seg, (a * (D2 * G + g.abs()))[:, None] * (o - pooled[seg]).abs())
    nb = torch.from_numpy(np.asarray(sizes, dtype=np.float64))[:, None]
    bound = 2 * U * ((nb + D2 + 8) * mag + spread)
    return dict(g=g, g_bound=(D2 + 2) * U * G, pooled=pooled, pooled_bound=bound)


def seg_sum_ref(gl, smax, sizes):
    """fp64 sum_n exp(gl_n - M) from the kernel's own fp32 gate logits and maximum, and its bound: n_b online-softmax steps, the
    8-warp merge and a few ulps of expf per term, plus the rounding of gl_n - M (u |gl_n - M| in the exponent)."""
    seg = segment_ids(sizes)
    gl64, M = gl.double(), smax.double()
    d = gl64 - M[seg]
    e = torch.exp(d)
    B = len(sizes)
    S = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, e)
    Sd = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, e * d.abs())
    nb = torch.from_numpy(np.asarray(sizes, dtype=np.float64))
    return S, 2 * U * ((nb + 12) * S + Sd)


def linear_ref(a, W, bias, relu: bool):
    """fp64 a @ W^T + bias (ReLU'd for a hidden layer) from the kernel's own fp32 input a, and the dot-product bound
    2 (K + 1) u (|a| |W|^T + |bias|).  ReLU is 1-Lipschitz, so the bound also covers a pre-activation near 0 that the kernel
    rounded to the other side."""
    a64, W64, b64 = a.double(), W.double(), bias.double()
    y = a64 @ W64.t() + b64
    bound = 2 * (W.shape[1] + 1) * U * (a64.abs() @ W64.abs().t() + b64.abs())
    return (torch.relu(y) if relu else y), bound


def readout_bwd_ref(h, x, w, sizes, dpooled, pooled, gl, smax, ssum, dw0, db0):
    """The readout gradients in fp64 from the kernel's own saved state (alpha_n = exp(gl_n - M_b) / S_b, pooled):
      dg_n = alpha_n (o_n . dp_b - pooled_b . dp_b),   d o_n = alpha_n dp_b + dg_n w,   dw_gate = dw0 + sum_n dg_n o_n,
      db_gate = db0 + sum_n dg_n
    (the chain rule of o -> softmax-weighted sum; tests/test_head_premises.py holds it to torch autograd) and their bounds,
    propagated to first order through alpha (expf, the subtraction, 1 / S: (|gl - M| + 6) u relative), the two length-2D dots
    o . dp and pooled . dp, the fmas of d o_n, and the summations of dw_gate / db_gate: per-warp chains of ceil(n_b / 8) rows, the
    8-warp merge, and B graph terms added to the accumulator in any order (atomics) or in graph order (deterministic mode).
    Every rounding may also land in fp32's subnormal range, with an absolute error of up to ETA = 2^-150 (an alpha of 1e-44 keeps
    only a few bits): that term is added wherever a value can be that small — alpha, dg_n and the products of d o_n."""
    seg = segment_ids(sizes)
    B = len(sizes)
    o = torch.cat([h, x], 1).double()
    D2 = o.shape[1]
    dp, p = dpooled.double(), pooled.double()
    w64 = w.double()
    d = gl.double() - smax.double()[seg]
    inv = 1.0 / ssum.double()[seg]
    alpha = torch.exp(d) * inv
    err_a = alpha * (d.abs() + 6) * U + ETA * (inv + 1)          # expf's and the product's subnormal rounding
    sd = (o * dp[seg]).sum(1)
    sd_mag = (o.abs() * dp.abs()[seg]).sum(1)
    cd, cd_mag = (p * dp).sum(1), (p.abs() * dp.abs()).sum(1)
    diff = sd - cd[seg]
    dg = alpha * diff
    E = alpha * (D2 + 6) * U * (sd_mag + cd_mag[seg]) + err_a * diff.abs() + U * dg.abs() + ETA
    do = alpha[:, None] * dp[seg] + dg[:, None] * w64
    do_bound = 2 * (err_a[:, None] * dp.abs()[seg] + E[:, None] * w64.abs() + 2 * U * (alpha[:, None] * dp.abs()[seg] + (dg[:, None] * w64).abs())
                    + 2 * ETA)
    chain = int(-(-int(np.max(sizes)) // READOUT_WARPS)) + READOUT_WARPS + B + 1
    dw = dw0.double() + (dg[:, None] * o).sum(0)
    dw_bound = 2 * ((E[:, None] * o.abs()).sum(0) + chain * U * ((dg.abs()[:, None] * o.abs()).sum(0) + dw0.double().abs())
                    + o.shape[0] * ETA)
    db = db0.double() + dg.sum()
    db_bound = 2 * (E.sum() + chain * U * (dg.abs().sum() + db0.double().abs()))
    D = D2 // 2
    return dict(dh=do[:, :D], dx=do[:, D:], dh_bound=do_bound[:, :D], dx_bound=do_bound[:, D:], dw=dw, dw_bound=dw_bound, db=db,
                db_bound=db_bound, seg=seg)


def mlp_bwd_ref(dlogits, pooled, acts, ws, dw0, db0):
    """ddfa_mlp_bwd in fp64 from its inputs: for i = L-1 .. 0, dW_i = dW0_i + dout^T in, db_i = db0_i + sum_rows dout,
    din = dout W_i (masked by in > 0 below layer 0), with bounds propagated through the layers — the bound of dout carried by
    |in| and |W_i|, plus the GEMM's own 2 (K + 1) u (|A| |B|) with K = B (weight and bias gradients) or the layer width (din).
    The mask is the kernel's (in > 0 of the fp32 activations it is given), so it is exact."""
    B = dlogits.shape[0]
    dout = dlogits.double()[:, None]
    bd = torch.zeros_like(dout)
    out = {}
    for i in range(len(ws) - 1, -1, -1):
        inp = (pooled if i == 0 else acts[i - 1]).double()
        W = ws[i].double()
        dW = dw0[i].double() + dout.t() @ inp
        dW_b = bd.t() @ inp.abs() + 2 * (B + 1) * U * (dout.abs().t() @ inp.abs() + dw0[i].double().abs())
        db = db0[i].double() + dout.sum(0)
        db_b = bd.sum(0) + 2 * (B + 1) * U * (dout.abs().sum(0) + db0[i].double().abs())
        din = dout @ W
        din_b = bd @ W.abs() + 2 * (W.shape[0] + 1) * U * (dout.abs() @ W.abs())
        out[i] = (dW, dW_b, db, db_b)
        if i > 0:
            mask = (inp > 0).double()
            dout, bd = din * mask, din_b * mask
        else:
            out["dpooled"] = (din, din_b)
    return out


def ratio(err, bound):
    """Largest err / bound (0 where both are 0, inf where only the bound is, nan where err is)."""
    err, bound = torch.as_tensor(err, dtype=torch.float64), torch.as_tensor(bound, dtype=torch.float64)
    if torch.isnan(err).any():
        return float("nan")
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return float(r.max()) if r.numel() else 0.0


# ---- graph loss -------------------------------------------------------------------------------------------------------------
def bce_sizes(B: int, seed: int) -> np.ndarray:
    """B graphs of 0-40 nodes, every 9th empty."""
    s = np.random.default_rng(seed).integers(1, 40, B)
    s[::9] = 0
    return s.astype(np.int64)


def bce_logits(B: int, seed: int) -> torch.Tensor:
    """randn * 4 with exact 0 and +-100 sprinkled in (exp(100) overflows fp32: the stable form must not)."""
    z = torch.randn(B, generator=torch.Generator().manual_seed(seed)) * 4
    z[3::11], z[5::13], z[7::17] = 0.0, 100.0, -100.0
    return z


# (num_graphs, num_valid): a full C1 batch with 24 padding graphs; nothing valid; B not a multiple of 8, with and without padding
BCE_CASES = [(1024, 1000), (13, 0), (1021, 1021), (37, 30)]


# ---- node-row sampler -------------------------------------------------------------------------------------------------------
_M0, _M1, _W0, _W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) in numpy uint64 arithmetic: ctr = 4 arrays (or ints) of 32-bit words, key = 2.
    Returns the 4 output words as uint64 arrays."""
    c = [np.asarray(v, dtype=np.uint64) & _MASK for v in ctr]
    k0, k1 = np.uint64(key[0]) & _MASK, np.uint64(key[1]) & _MASK
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = _M0 * c[0], _M1 * c[2]                  # 32 x 32 -> 64 bits: exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return c


def node_keys(N: int, seed: int, draw: int) -> np.ndarray:
    """The sampler's key of every node: word 0 of Philox4x32-10, key = seed, counter (draw lo, draw hi, node, 0)."""
    n = np.arange(N, dtype=np.uint64)
    z = np.zeros(N, dtype=np.uint64)
    return philox4x32_10((z + np.uint64(draw & 0xFFFFFFFF), z + np.uint64((draw >> 32) & 0xFFFFFFFF), n, z),
                         (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))[0]


def sample_ref(vuln, num_valid: int, factor: float, seed: int, draw: int):
    """What ddfa_node_sample promises (include/ddfa_b200.h): (rows, num_rows, overflow, next draw).  factor < 0: every valid node,
    the draw is not used.  Otherwise every valid vulnerable node plus the k = rint(n_vuln * factor) smallest (key, node) pairs of
    the valid non-vulnerable ones (all of them, and overflow = True, when k exceeds their number), in ascending node order."""
    vuln = np.asarray(vuln)
    N = len(vuln)
    nv = min(max(int(num_valid), 0), N)
    if factor < 0:
        return np.arange(nv, dtype=np.int32), nv, False, draw
    v = vuln[:nv] != 0
    pop = np.nonzero(~v)[0]
    want = np.rint(float(np.count_nonzero(v)) * factor)
    overflow = not (want <= len(pop))
    k = len(pop) if overflow else int(want)
    keys = node_keys(nv, seed, draw)[pop]
    take = pop[np.lexsort((pop, keys))[:k]]            # by key, then by node
    rows = np.sort(np.concatenate([np.nonzero(v)[0], take])).astype(np.int32)
    return rows, len(rows), overflow, draw + 1


@functools.lru_cache(maxsize=None)
def tie_case():
    """A C1-size sampler draw whose k-th smallest key is shared by two nodes a < b in different sampler CTAs.  On the C1 batch's
    vuln (with a and b made non-vulnerable), draw 0, the first seed with such a pair whose key no other node has; factor_a makes
    k = (#non-vulnerable nodes below the key) + 1, so only a is taken, factor_ab one more, so both are."""
    g = c1_batch()
    vuln = g.ndata["_VULN"].numpy().astype(np.int32).copy()
    N = len(vuln)
    for seed in range(64):
        keys = node_keys(N, seed, 0)
        order = np.argsort(keys, kind="stable")
        ks = keys[order]
        dup = np.nonzero(ks[1:] == ks[:-1])[0]
        for i in dup:
            a, b = int(order[i]), int(order[i + 1])
            if (i > 0 and ks[i - 1] == ks[i]) or (i + 2 < N and ks[i + 2] == ks[i]) or a // SAMPLER_CTA_NODES == b // SAMPLER_CTA_NODES:
                continue
            v = vuln.copy()
            v[[a, b]] = 0
            n_vuln = int(np.count_nonzero(v))
            below = int(np.count_nonzero((keys < ks[i]) & (v == 0)))
            fa, fab = (below + 1) / n_vuln, (below + 2) / n_vuln
            return dict(seed=seed, a=a, b=b, key=int(ks[i]), vuln=v, n_vuln=n_vuln, below=below, factor_a=fa, factor_ab=fab,
                        k_a=undersample_count(n_vuln, fa), k_ab=undersample_count(n_vuln, fab))
    return None


def sampler_cases():
    """(name, vuln, num_valid, factor, seed, draw) of the GPU sampler test; the premises file checks each reaches its edge."""
    rng = np.random.default_rng(77)
    cases = []
    v = (rng.random(5000) < 0.3).astype(np.int32)
    cases.append(("ragged_N", v, 5000, 1.0, 3, 0))                              # 5 CTAs, the last one 904 nodes
    cases.append(("N1_clean", np.zeros(1, np.int32), 1, 1.0, 1, 0))            # n_vuln = 0: k = 0, no rows
    cases.append(("N1_vuln", np.ones(1, np.int32), 1, 2.0, 1, 0))              # k = 2 > population 0: status, one row
    cases.append(("N1_clean_all", np.zeros(1, np.int32), 1, 1e6, 1, 0))
    cases.append(("num_valid_0", (rng.random(3000) < 0.5).astype(np.int32), 0, 1.0, 2, 5))
    v = (rng.random(6000) < 0.2).astype(np.int32)
    v[4321:] = 1                                                                # vulnerable padding nodes
    cases.append(("padding", v, 4321, 1.5, 4, 9))
    v = (rng.random(4100) < 0.1).astype(np.int32)
    cases.append(("k0", v, 4100, 0.0, 5, 0))
    pop = int(np.count_nonzero(v == 0))
    cases.append(("k_pop", v, 4100, pop / int(np.count_nonzero(v)), 5, 1))    # exactly the population, no status
    cases.append(("k_over", v, 4100, 1e9, 5, 2))                               # status, the whole population
    cases.append(("all_rows", v, 3333, -1.0, 5, 3))                            # no undersampling: every valid node
    for nv_, f in ((5, 0.5), (7, 0.5), (3, 1.5)):                               # 2.5 -> 2, 3.5 -> 4, 4.5 -> 4
        v = np.zeros(2500, np.int32)
        v[rng.choice(2500, nv_, replace=False)] = 1
        cases.append((f"half_{nv_}x{f}", v, 2500, f, 6, 0))
    v = (rng.random(9000) < 0.05).astype(np.int32)
    cases.append(("draw_hi", v, 9000, 2.0, 7, (3 << 32) + 5))                   # the draw's high word is used
    g = c1_batch()
    cases.append(("c1", g.ndata["_VULN"].numpy().astype(np.int32), g.num_nodes(), 1.0, 11, 40))
    t = tie_case()
    cases.append(("c1_tie_a", t["vuln"], len(t["vuln"]), t["factor_a"], t["seed"], 0))
    cases.append(("c1_tie_ab", t["vuln"], len(t["vuln"]), t["factor_ab"], t["seed"], 0))
    return cases


# ---- node-style head (node_loss.cu: ddfa_node_head_fwd / _bwd) ----------------------------------------------------------------
NODE_HEAD_BM, NODE_HEAD_BK = 64, 16     # head_gemm_kernel: 64-row tiles, K in steps of 16 (a ragged last step when 2D % 16 != 0)
NODE_HEAD_CHUNKS = 32                   # kHeadChunks: row chunks of the weight / bias gradient, added in chunk order
NODE_HEAD_WARP_ROWS = 8                 # head_out_kernel: a warp per row, 8 rows per CTA
NODE_HEAD_WIDTHS = (20, 32, 64, 128, 192, 256, 320, 384, 448, 512)    # D: the SIMT widths and the tensor-core wide widths
NODE_SMALL_S = (0, 1, 5, 31, 32, 33, -1)                              # row counts at the hub node count; -1: every node
NODE_VULN_RATE, NODE_FACTOR = 0.15, 1.0                               # the C1 row list: every vulnerable node + as many others


def node_head_chunks(S: int):
    """The rows [r0, r1) of each weight-gradient chunk (head_wgrad_kernel / head_bias_partial_kernel): ceil(S / 32) rows each."""
    c = -(-S // NODE_HEAD_CHUNKS)
    return [(min(S, i * c), min(S, min(S, i * c) + c)) for i in range(NODE_HEAD_CHUNKS)]


def node_head_ws_bytes(N: int, D: int) -> int:
    """ddfa_node_head_bwd_workspace_bytes: two [N, 2D] planes and 32 chunk partials of a [2D, 2D] gradient plus its bias."""
    K = 2 * D
    return 4 * (2 * N * K + NODE_HEAD_CHUNKS * (K * K + K))


def node_rows_trainer(N: int, seed: int) -> np.ndarray:
    """A row list as FusedTrainer draws it (sample_ref: every vulnerable node plus rint(n_vuln * factor) non-vulnerable ones by
    Philox key), over NODE_VULN_RATE labels with node 0 and node N - 1 vulnerable, so both ends of the planes are in it."""
    vuln = (np.random.default_rng(seed).random(N) < NODE_VULN_RATE).astype(np.int32)
    vuln[[0, N - 1]] = 1
    return sample_ref(vuln, N, NODE_FACTOR, seed, 0)[0]


def node_rows(N: int, S: int, seed: int) -> np.ndarray:
    """S sorted unique rows of N (S < 0: all of them); node N - 1 first, then node 0, then random ones."""
    if S < 0 or S >= N:
        return np.arange(N, dtype=np.int32)
    fixed = [N - 1, 0][:S]
    rest = np.random.default_rng(seed).choice(np.arange(1, N - 1), max(S - len(fixed), 0), replace=False)
    return np.sort(np.concatenate([fixed, rest])).astype(np.int32)


def node_head_ref(ins0, acts, ws, bs, dl, dw0, db0):
    """The node head's forward and backward in float64 from the kernel's own fp32 inputs to each stage, with every hidden ReLU on
    the side of its kink the kernel's forward took (mask = act > 0): the autograd of [h | x][rows] -> Linear/ReLU ... ->
    Linear(2D, 1) with relu(z) read as z * mask.  ins0: [S, 2D] gathered rows; acts: the kernel's hidden activations [S, 2D]
    each; dl: [S] dlogits; dw0 / db0: the gradients' start values (the kernel accumulates).

    Returns name -> (ref, mag, tau) with |got - ref| <= tau * mag the a-priori bound of each output (u = 2^-24, every count
    doubled as in linear_ref): mag is the same computation on absolute values.  Forward: a length-(K + 1) dot product
    (2 (K + 1) u).  Backward: the error of the incoming gradient (its own tau, carried by the absolute-value chain) plus, for
    dIn, a length-K dot product (or one product for the last layer), and for dW / db a ceil(S / 32)-row chunk sum, the 32-way
    chunk reduction and the add onto the start value (2 (ceil(S / 32) + 34) u)."""
    L = len(ws)
    K = ins0.shape[1]
    S = ins0.shape[0]
    chunk = -(-S // NODE_HEAD_CHUNKS)
    f64 = lambda t: t.double()
    ins = [f64(ins0)] + [f64(a) for a in acts]
    masks = [f64(a > 0) for a in acts]
    out = {}
    fwd_tau = 2 * (K + 1) * U
    for i in range(L):
        W, b = f64(ws[i]), f64(bs[i])
        z = ins[i] @ W.t() + b
        mag = ins[i].abs() @ W.abs().t() + b.abs()
        if i < L - 1:
            out[f"act{i}"] = (torch.relu(z), mag, fwd_tau)
        else:
            out["logits"] = (z[:, 0], mag[:, 0], fwd_tau)
    g, gmag, gtau = f64(dl)[:, None], f64(dl).abs()[:, None], 0.0
    w_tau = 2 * (chunk + 34) * U
    for i in range(L - 1, -1, -1):
        W = f64(ws[i])
        dw = g.t() @ ins[i] + f64(dw0[i])
        dwm = gmag.t() @ ins[i].abs() + f64(dw0[i]).abs()
        out[f"dw{i}"] = (dw, dwm, gtau + w_tau)
        out[f"db{i}"] = (g.sum(0) + f64(db0[i]), gmag.sum(0) + f64(db0[i]).abs(), gtau + w_tau)
        step = 2 * U if i == L - 1 else 2 * (K + 1) * U          # dlogits[s] * w[k] (one product) or a length-K dot product
        g, gmag, gtau = g @ W, gmag @ W.abs(), gtau + step
        if i > 0:
            g, gmag = g * masks[i - 1], gmag * masks[i - 1]
    out["din"] = (g, gmag, gtau)
    return out
