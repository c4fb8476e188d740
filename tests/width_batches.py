"""Hidden widths of the SIMT engine and the launch formulas of the kernels it runs, shared by tests/test_width_gpu.py (which runs
the kernels at these widths and sizes) and tests/test_width_premises.py (which checks, without a GPU, that the shapes still reach
every dispatch path the GPU tests are written for).

Every formula below restates the host code of one kernel: sgemm() and sgemm_splitk_ordered_slices() (csrc/sgemm.cu),
simt_wgrad_split() and the gru_gate_bwd_kernel launch (csrc/gru_step.cu), ddfa_gather_sum (csrc/gather.cu), the default and
deterministic embedding backward launches (csrc/embed.cu)."""
from scale_batches import HUB_SHAPES, NUM_SMS

# W -> (K tables, H columns per table): W = K * H is the row width of the embedding and the hidden width of the GatedGraphConv.
# K = 4 is concat_all_absdf=True with hidden_dim = H, K = 1 is a single table of hidden_dim = H.
WIDTHS = {
    20: (1, 20),      # gather G = 8 with 3 idle lanes; gate backward block (5, 51); H / 4 = 5 is not a power of two
    32: (1, 32),      # the reference's hidden_dim without concat; 3W = 96 is below one 128-column tile
    48: (4, 12),      # deterministic embedding TL = 4 (H / 4 = 3); W not a multiple of 32
    64: (4, 16),      # small concat width
    96: (4, 24),      # gather G = 32, CH = 1 at a width other than 128; 3W = 288: a ragged third tile
    128: (1, 128),    # a single 128-wide table: the image embedding; both engines
    256: (4, 64),     # gather CH = 2; 3W = 768
    512: (1, 512),    # the widest the module runs: deterministic embedding COLS = 4, fold on the 128x128 kernel, gather CH = 4
}
MAX_WIDTH = 512       # readout.cu kMaxChunks * 128 and the embedding backward's K * H <= 512

C1_NODES = HUB_SHAPES["c1"][2]      # 157 381: the node count of the sgemm, embedding and GRU step tests
EMBED_V = 1002                      # the reference's input_dim

# ---- csrc/sgemm.cu -------------------------------------------------------------------------------------------------------
BK = 16              # k depth of one 128x128 tile step (the ordered split-K slices are whole multiples of it)
SMALL_MAX_MN = 512 * 512
SMALL_MAX_K = 4096


def sgemm_plan(M: int, N: int, K: int, beta: float = 0.0, split_k: int = 1, deterministic: bool = False) -> dict:
    """Which kernel sgemm() launches, its z-slices, and the summation depth of one output element: the length of the fp32 FMA
    chain of one slice plus the number of slice sums added into C (the a-priori error bound of the GPU tests is depth * u)."""
    split_k = max(1, split_k)
    if split_k == 1 and M * N <= SMALL_MAX_MN and K <= SMALL_MAX_K:
        tiles = -(-N // 32) * -(-M // 32)
        split = 1
        if beta == 1.0 and K >= 256 and tiles < NUM_SMS and not deterministic:
            split = max(1, min((2 * NUM_SMS + tiles - 1) // tiles, K // 64))
        kps = max(32, (-(-K // split) + 31) // 32 * 32)
        z = -(-K // kps) if K > kps else 1
        return dict(kernel="small", tiles=tiles, z=z, kps=kps, atomic=z > 1, depth=min(K, kps) + z)
    k_tiles = -(-K // BK)
    if split_k > k_tiles:
        split_k = k_tiles if k_tiles > 0 else 1
    kps = -(-k_tiles // split_k) * BK
    if split_k > 1 and deterministic:
        return dict(kernel="refused")
    return dict(kernel="big", tiles=-(-N // 128) * -(-M // 128), z=split_k, kps=kps, atomic=split_k > 1, depth=min(K, kps) + split_k)


def ordered_plan(K: int, split_k: int) -> dict:
    """sgemm_splitk_ordered (the deterministic weight gradient): nz slices of kps rows, the last one kps or shorter, each slice
    written to its own block and the blocks added in order by splitk_reduce_kernel."""
    k_tiles = -(-K // BK)
    split_k = max(1, min(split_k, k_tiles))
    kps = -(-k_tiles // split_k) * BK
    nz = -(-K // kps) if K > 0 else 1
    return dict(nz=nz, kps=kps, last=K - (nz - 1) * kps, depth=min(K, kps) + nz)


def simt_wgrad_split(N: int, D: int) -> int:
    tiles = -(-3 * D // 128) * -(-D // 128)
    split = (2 * NUM_SMS + tiles - 1) // tiles
    k_tiles = -(-N // 16)
    if split > k_tiles // 8:
        split = k_tiles // 8 if k_tiles // 8 > 0 else 1
    return split


def engine_sgemm_calls(W: int, N: int) -> dict:
    """The sgemm calls of one SIMT GRU step, the weight fold and the batched MLP head for hidden width W and N nodes:
    name -> (ta, tb, M, N, K, beta, split_k).  The head runs on rows of 2W (B = 1024 graphs, the C1 batch)."""
    D2, B = 2 * W, 1024
    return {
        "fwd gi/gh": (0, 1, N, 3 * W, W, 0.0, 1),
        "dgrad ds": (0, 0, N, W, 3 * W, 0.0, 1),
        "dgrad dh": (0, 0, N, W, 3 * W, 1.0, 1),
        "wgrad": (1, 0, 3 * W, W, N, 1.0, simt_wgrad_split(N, W)),
        "fold fwd": (0, 0, 3 * W, W, W, 0.0, 1),
        "fold bwd dW_ih": (0, 1, 3 * W, W, W, 1.0, 1),
        "fold bwd dW": (1, 0, W, W, 3 * W, 1.0, 1),
        "head fwd": (0, 1, B, D2, D2, 0.0, 1),
        "head wgrad": (1, 0, D2, D2, B, 1.0, 1),
        "head dgrad": (0, 0, B, D2, D2, 0.0, 1),
    }


# Shapes just either side of each dispatch boundary of sgemm(): name -> (ta, tb, M, N, K, alpha, beta)
SGEMM_EDGES = {
    "mn=512^2": (0, 0, 512, 512, 96, 1.0, 0.0),
    "mn=512^2+1": (0, 0, 5, 52_429, 96, 1.0, 0.0),          # 5 * 52 429 = 512^2 + 1
    "mn=512x513": (0, 1, 512, 513, 96, 1.0, 0.0),            # one more column
    "k=4096": (1, 0, 64, 64, 4096, 1.0, 0.0),
    "k=4097": (1, 0, 64, 64, 4097, 1.0, 0.0),
    "k=255,beta=1": (1, 0, 64, 64, 255, 1.0, 1.0),
    "k=256,beta=1": (1, 0, 64, 64, 256, 1.0, 1.0),
    "tiles=131": (1, 0, 32, 131 * 32, 512, 1.0, 1.0),
    "tiles=132": (1, 0, 4 * 32, 33 * 32, 512, 1.0, 1.0),
    "small,alpha,beta=0.5": (0, 1, 96, 300, 200, -0.75, 0.5),
    "big,alpha,beta=0.5": (0, 1, 700, 520, 200, -0.75, 0.5),
    "big,beta=1": (1, 1, 600, 500, 1000, 1.5, 1.0),
}

# ---- csrc/gather.cu: ddfa_gather_sum's instance for D != 128 ----------------------------------------------------------------
def gather_instance(D: int):
    """(G lanes per row group, CH 16-byte chunks per lane) of gather_sum_kernel for width D; "d128" for the tuned D = 128 set."""
    chunks = D // 4
    if D == 128:
        return "d128"
    for limit, inst in ((8, (8, 1)), (16, (16, 1)), (32, (32, 1)), (64, (32, 2)), (128, (32, 4))):
        if chunks <= limit:
            return inst
    return (32, 8)


# ---- csrc/gru_step.cu: gru_gate_bwd_kernel ----------------------------------------------------------------------------------
GATE_BWD_ROWS = 128                 # kGateBwdRows


def gate_bwd_launch(N: int, D: int) -> dict:
    bx = D // 4
    by = 256 // bx if 256 // bx > 0 else 1
    return dict(block=(bx, by), ctas=-(-N // GATE_BWD_ROWS), smem=4 * by * 7 * D, rows_per_thread=-(-GATE_BWD_ROWS // by))


# ---- csrc/embed.cu ---------------------------------------------------------------------------------------------------------
EMB_ROWS = 256                      # kEmbRows: node rows per CTA of the default backward
DET_CHUNK = 256                     # kDetChunk: sorted positions per team of the deterministic backward


def embed_bwd_launch(N: int, K: int, H: int) -> dict:
    D = K * H
    bx = D // 4
    by = 256 // bx if 256 // bx > 2 else 2
    return dict(block=(bx, by), ctas=-(-N // EMB_ROWS), smem=4 * by * 2 * D)


def embed_det_launch(N: int, H: int) -> dict:
    hq = H // 4
    TL = 1
    while TL < hq and TL < 32:
        TL *= 2
    return dict(TL=TL, COLS=1 if hq <= 32 else 4, chunks=-(-N // DET_CHUNK))


def embed_depth(N: int) -> int:
    """Summation depth of one embedding-gradient element, both paths: at most a CTA's (default) or a chunk's (deterministic)
    256 rows in one chain, then one partial per CTA / chunk (plus the deterministic combine's 8-way tree), the dx + dx2 add and
    the add into the table."""
    return EMB_ROWS + -(-N // EMB_ROWS) + 8 + 2
