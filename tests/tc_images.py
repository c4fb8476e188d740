"""Host decoders of the tensor-core engine's device formats — the activation image and the packed saved gates — shared by
tests/test_kernels_gpu.py and tests/test_scale_gpu.py."""
import torch


def decode_image(img: torch.Tensor, N: int) -> torch.Tensor:
    """Activation image (include/ddfa_b200.h) -> fp64 [N,128] = hi + lo, undoing the SWIZZLE_128B unit permutation."""
    tiles = img.numel() // 65536
    raw = img.cpu().view(torch.int16).view(tiles, 4, 128, 8, 8)                   # [tile][chunk = 2 v + kb][row][physical 16-B unit][8 bf16]
    rows = torch.arange(128).view(1, 1, 128, 1, 1)
    units = torch.arange(8).view(1, 1, 1, 8, 1)
    phys = (units ^ (rows & 7)).expand(tiles, 4, 128, 8, 8)
    logical = torch.gather(raw, 3, phys)                                          # logical unit j sits at physical unit j ^ (row & 7)
    vals = (logical.to(torch.int32) << 16).view(torch.float32).double().view(tiles, 2, 2, 128, 64)   # [tile][v][kb][row][col in block]
    x = (vals[:, 0] + vals[:, 1]).permute(0, 2, 1, 3).reshape(tiles * 128, 128)   # hi + lo, [row][kb][64] -> 128 columns
    assert float(x[N:].abs().max()) == 0.0 if x.shape[0] > N else True           # rows past N are zero
    return x[:N]


def decode_gates(gates: torch.Tensor, N: int):
    """Packed saved gates (csrc/tc_common.cuh: pack_gates) -> (r, z, n, gh_n) fp64 [N,128]."""
    w = gates.cpu().view(torch.int32).view(N, 128, 2).to(torch.int64) & 0xffffffff
    x, y = w[..., 0], w[..., 1]
    r = (x & 0x3fff).double() / 16383.0
    z = ((x >> 14) & 0x3fff).double() / 16383.0
    nq = y & 0xffff
    n = torch.where(nq >= 32768, nq - 65536, nq).double() / 32767.0
    g = ((y >> 16) << 4) | (x >> 28)
    e, m, sign = (g >> 14) & 31, (g & 0x3fff).double(), (g >> 19) & 1
    ghn = torch.where(e == 0, torch.zeros_like(m), torch.pow(2.0, (e - 15).double()) * (1.0 + m / 16384.0))
    return r, z, n, torch.where(sign == 1, -ghn, ghn)
