"""Widths and launch shapes of the tensor-core engine above 128 (csrc/gru_tc_wide.cu), shared by tests/test_wide_tc_gpu.py (which runs
the GEMMs at these widths on the C1 node count) and tests/test_wide_tc_cpu.py (which checks, without a GPU, that those shapes reach
every tail case of the kernel).

Every formula restates the host code of gru_tc_wide.cu: tcw_gemm() (the grid: 128 x 128 output tiles, n tile fastest, then m tile,
then split-K slice; K in steps of 64), tcw_wgrad_split() and tcw_slices() (the weight gradient's slices over K = nodes)."""
from scale_batches import NUM_SMS

WIDE_WIDTHS = (192, 256, 320, 384, 448, 512)      # the multiples of 64 from 192 to the module's maximum
TILE, KSTEP = 128, 64
MAX_SPLIT = 32


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def wgrad_split(N: int, D: int) -> int:
    """tcw_wgrad_split: the slice count s <= 32 whose tiles x s CTAs fill their last wave best (smallest s on a tie), at most one
    slice per 64-node step."""
    tiles = cdiv(3 * D, TILE) * cdiv(D, TILE)
    nks = cdiv(N, KSTEP)
    best, best_fill = 1, (0, 1)
    for s in range(1, MAX_SPLIT + 1):
        ctas = tiles * s
        den = cdiv(ctas, NUM_SMS) * NUM_SMS
        if ctas * best_fill[1] > best_fill[0] * den:
            best, best_fill = s, (ctas, den)
    return best if best < nks else max(nks, 1)


def wgrad_slices(N: int, D: int) -> dict:
    """tcw_slices: kps 64-node steps per slice, nz slices, the last one `last` steps long."""
    nks = cdiv(N, KSTEP)
    kps = max(1, cdiv(nks, wgrad_split(N, D)))
    nz = cdiv(nks, kps) if nks > 0 else 1
    return dict(nks=nks, kps=kps, nz=nz, last=nks - (nz - 1) * kps)


def gemm_launches(N: int, D: int) -> dict:
    """The three GEMM shapes of one step (forward, dgrad, weight gradient): M, N, K, the output tiles, whether the last m / n tile
    has only one valid 64-wide half, the K steps (odd / even) and the CTAs of the launch."""
    out = {}
    for name, (M, Nn, K) in {"fwd": (N, 3 * D, D), "dgrad": (N, D, 3 * D), "wgrad": (3 * D, D, N)}.items():
        nks = cdiv(K, KSTEP)
        nz = wgrad_slices(N, D)["nz"] if name == "wgrad" else 1
        out[name] = dict(M=M, N=Nn, K=K, m_tiles=cdiv(M, TILE), n_tiles=cdiv(Nn, TILE), m_half=M % TILE == KSTEP,
                         n_half=Nn % TILE == KSTEP, m_ragged=M % TILE, nks=nks, ctas=cdiv(M, TILE) * cdiv(Nn, TILE) * nz)
    return out
