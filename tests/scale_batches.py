"""Hub batches and the launch shapes of the tensor-core kernels, shared by tests/test_scale_gpu.py (which runs the kernels at these
shapes) and tests/test_scale_premises.py (which checks, without a GPU, that the shapes still reach the trip counts the GPU tests
are written for)."""
import functools

import numpy as np
import torch

from deepdfa_b200 import batched_graph as G
from deepdfa_b200 import synth

# Launch formulas of csrc/gru_tc_bwd.cu and csrc/gru_tc_fwd3.cu (H100: kNumSMs = 132)
NUM_SMS = 132
TILE = 128                  # rows per activation-image tile (tcc::kTileM)
GATE_BWD_ROWS = 32          # rows per gate-backward block (tc2b::kGtRows)
GATE_BWD_STAGES = 3         # tc2b::kGtStages: a CTA refills a stage only when it owns more blocks than this
GEMM_GROUPS = NUM_SMS // 4  # gru_fwd3_kernel (4 column slices) and dgrad3_kernel (2 roles x 2 column halves)
WGRAD_CTAS = NUM_SMS // 6   # kWgCtas: x 6 gate blocks = one CTA per SM
WGRAD_MAX_STEPS = 16        # DDFA_WGRAD_MAX_STEPS: above it the weight gradient is accumulated step by step


def trip_counts(N: int, steps: int = 1) -> dict:
    """Per-CTA trip counts of the persistent tensor-core kernels for N nodes (least loaded CTA / most loaded CTA)."""
    tiles = -(-N // TILE)
    blocks = tiles * TILE // GATE_BWD_ROWS
    gb_grid = min(blocks, NUM_SMS)
    groups = min(GEMM_GROUPS, tiles)
    wg_tiles = tiles * steps
    return dict(tiles=tiles, gate_bwd_blocks=(blocks // gb_grid, -(-blocks // gb_grid)),
                gemm_tiles=(tiles // groups, -(-tiles // groups)), wgrad_tiles=(wg_tiles // WGRAD_CTAS, -(-wg_tiles // WGRAD_CTAS)))


# Rows (local to the hub graph) and the in-degrees they are given.  33 / 64 / 65 cross the 32-id prefetch window of the image
# gathers and TMA variants and NIDX*G = 64 of register variants 2/3/5; 200 and the last row's 1100 wrap the 16-row TMA ring many times.
HUB_IN = {10: 33, 20: 64, 30: 65, 40: 200}
LAST_HUB_IN = 1100
GROUP_IN = (40, 33, 90, 17)           # four consecutive rows of one 4-row warp group
ZERO_IN, ZERO_OUT = (5, 6), (7, 8)    # no in-edge at all (not even a self-loop) / no out-edge
OUT_HUB = (60, 1000)                  # one row with 1000 out-edges: a 1000-neighbour row of the transposed CSR
OUT_WIDE = range(70, 80)              # out-degree 8, 11, ..., 35: transposed in-degree above the folded-gather prefetch (4 / 2)


def make_hub_batch(num_graphs: int, seed: int, target_nodes: int) -> G.BatchedCFG:
    """``synth.make_batch(num_graphs, 150, variable=True)`` plus one last graph of ``target_nodes - N`` nodes that holds the hubs:
    the rows of HUB_IN, four consecutive hub rows inside one warp group, a 1100-neighbour hub as the very last row N-1 (in a
    ragged last 128-row tile), wide out-degrees, rows without in-edges or out-edges, and duplicate edges."""
    base = synth.make_batch(num_graphs, 150, seed=seed, variable=True, vuln_rate=0.3)
    off = base.num_nodes()
    H = target_nodes - off
    assert H >= 1300, H
    hub = synth.make_batch(sizes=[H], seed=seed + 1, vuln_rate=1.0)
    src, dst = [t.numpy().copy() for t in hub.edges()]
    rng = np.random.default_rng(seed)
    g0 = 100 + (-(off + 100)) % 4                  # first row of the warp group: global id divisible by 4
    in_deg = dict(HUB_IN)
    in_deg.update({g0 + i: d for i, d in enumerate(GROUP_IN)})
    in_deg[H - 1] = LAST_HUB_IN
    fixed = list(in_deg) + list(ZERO_IN)           # rows whose in-edges are exactly the ones added below
    keep = ~np.isin(dst, fixed) & ~np.isin(src, ZERO_OUT)
    src, dst = [src[keep]], [dst[keep]]
    pool = np.setdiff1d(np.arange(H), ZERO_OUT)
    free = np.setdiff1d(np.arange(H), fixed)
    for row, d in in_deg.items():                  # sources drawn with replacement: duplicate edges
        src.append(rng.choice(pool, d)); dst.append(np.full(d, row))
    src.append(np.full(OUT_HUB[1], OUT_HUB[0])); dst.append(rng.choice(free, OUT_HUB[1]))
    for i, u in enumerate(OUT_WIDE):
        src.append(np.full(8 + 3 * i, u)); dst.append(rng.choice(free, 8 + 3 * i))
    src.append(np.array([11, 11, 11])); dst.append(np.array([12, 12, 12]))   # a triple edge
    hub = G.BatchedCFG(torch.from_numpy(np.concatenate(src)), torch.from_numpy(np.concatenate(dst)), hub.batch_num_nodes(), hub.ndata)
    return G.batch([base, hub])


# name -> (make_hub_batch arguments, what the GPU tests rely on at that size)
HUB_SHAPES = {
    "threshold": (66, 900, 12_701),     # 400 gate-backward blocks: CTAs 0-3 own 4 and refill one stage once
    "mid": (252, 41, 40_001),           # the whole GatedGraphConv, T = 8 (batched weight gradient) and T = 17 (per step)
    "c1": (1016, 32, 157_381),          # about the benchmark's C1 batch (make_batch(1024, 150, variable=True): 157 377 nodes)
}


MODULE_C1 = dict(num_graphs=1024, nodes_per_graph=150, seed=11, variable=True, vuln_rate=0.3)    # the module-gradient batch at C1


@functools.lru_cache(maxsize=None)
def hub_batch(name: str) -> G.BatchedCFG:
    return make_hub_batch(*HUB_SHAPES[name])


def degrees(g):
    src, dst = [t.numpy() for t in g.edges()]
    N = g.num_nodes()
    return np.bincount(dst, minlength=N), np.bincount(src, minlength=N)
