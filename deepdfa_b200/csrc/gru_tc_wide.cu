// Tensor-core engine at the wide hidden widths (D = 192 .. 512, D % 64 == 0): the six dense GEMMs of one GRU step on Hopper
// warpgroup MMA (wgmma), with the SIMT engine's data flow around them (fp32 row-major planes, gru_gate_fwd_kernel /
// gru_gate_bwd_kernel, the four fp32 saved-gate planes; gru_step.cu).
//
// Arithmetic is the D = 128 engine's: every operand is split into bf16 hi = bf16(x) and lo = bf16(x - hi), each product is
// hi*hi + hi*lo + lo*hi with fp32 accumulation, and every operand is kept as an image (tc_common.cuh: image_offset_w) — 128-row
// tiles of [hi | lo][D / 64 column chunks], each chunk [128 rows x 64 bf16] in the K-major SWIZZLE_128B layout.  An image serves
// two ways: read K-major, its rows are the M (or N) rows of the product and its columns the K dimension; read MN-major
// (transposed), its rows are K and its columns M (or N).  So one image per matrix covers all three GEMMs:
//
//   call                    M        N     K        A (rows x K)               B (N x K)
//   gi = s W'^T, gh = h Whh^T  nodes  3D    D        s / h image, K-major        W' / Whh image, K-major
//   ds = dgi W', dh += dgh Whh nodes  D     3D       dgi / dgh image, K-major    W' / Whh image, MN-major
//   dW' += dgi^T s, dWhh ...   3D     D     nodes    dgi / dgh image, MN-major   s / h image, MN-major
//
// One kernel, templated on the two operand majors.  A CTA computes a [128 x 128] tile of C over a range of K (the whole K, or
// one split-K slice of the weight gradient) in steps of 64: a producer warp streams each step's A and B hi / lo into a ring of
// three 64 KB stages with 1-D TMA bulk copies; two consumer warpgroups own rows 0-63 / 64-127 (m64n128k16).  Each step (K = 64)
// is accumulated in the MMA registers and then added to a running fp32 sum with ordinary adds: the tensor core's
// accumulation does not round to nearest, and chaining all of K in it biases long sums toward zero (gru_tc_bwd.cu,
// wgrad_kernel).
//
// Tails.  Every D here is a multiple of 64, so a 128-wide tile of 3D or D columns is either full or has exactly one valid
// 64-column half: an MN-major operand copies only the valid half (the other half of the stage keeps stale data, which reaches
// only output columns that are never stored), and a K-major weight image is padded with zero rows to a whole tile.  Node rows
// past N are zero in every image (to_image_kernel), so they add nothing to a K = nodes sum, and no output row past N is stored.
//
// The weight gradient is split over K = nodes into slices (tcw_wgrad_split) that each write a private [3D x D] block; one
// kernel then adds the blocks to dW in slice order, in both modes — the sum is the same bit for bit on every run.
#include "tc_common.cuh"

namespace ddfa {
namespace tcw {
using namespace tcc;

constexpr int kBM = 128, kBN = 128, kBK = 64;
constexpr int kStages = 3;
constexpr int kOpBytes = 2 * kChunkBytes;                 // one operand of one step: [hi | lo] x 16 KB
constexpr int kStageBytes = 2 * kOpBytes;                 // A then B: 64 KB
constexpr int kOffBar = kStages * kStageBytes;
constexpr int kSmemAlloc = kOffBar + 2 * kStages * 8 + 1024;      // + slack to align the window to 1024 bytes (SWIZZLE_128B)
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 32;        // two consumer warpgroups + one producer warp
static_assert(kSmemAlloc <= 232448, "shared memory budget");

// one GEMM operand: an image (tc_common.cuh: image_offset_w) of a matrix with `cols` columns, cols % 64 == 0
struct Operand {
  const uint8_t *img;
  int32_t cols;
};

__device__ __forceinline__ size_t chunk_at(const Operand &op, int tile, int v, int kb) {
  return (size_t)tile * ((size_t)kTileM * 4 * op.cols) + (size_t)(v * (op.cols >> 6) + kb) * kChunkBytes;
}

// Issue the copies of one operand for K step ks into the stage region `dst` ([hi | lo], 16 KB each) and return their bytes.
//   K-major (MN == 0): the operand's 128 rows r0 .. r0 + 127 = one image tile, K columns 64 ks .. 64 ks + 63 = its chunk ks.
//   MN-major (MN == 1): K rows 64 ks .. 64 ks + 63 = half an image tile (8 KB of each chunk), the 128 M / N columns r0 .. = two
//   chunks, the second only if it exists; each 64-column half lands 8 KB apart.
template <int MN>
__device__ __forceinline__ uint32_t operand_bytes(const Operand &op, int r0) {
  if (MN == 0) return kOpBytes;
  return ((r0 >> 6) + 1 < (op.cols >> 6) ? 2u : 1u) * 2u * 8192u;
}
template <int MN>
__device__ __forceinline__ void copy_operand(const Operand &op, int r0, int ks, uint32_t dst, uint32_t bar) {
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    if (MN == 0) {
      bulk_g2s(dst + v * kChunkBytes, op.img + chunk_at(op, r0 / kTileM, v, ks), kChunkBytes, bar);
    } else {
      const int k0 = ks * kBK;
      const size_t row_off = (size_t)(k0 % kTileM) * 128;      // 64 swizzled 128-byte rows, 8-row groups stay whole
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int kb = (r0 >> 6) + j;
        if (kb < (op.cols >> 6))
          bulk_g2s(dst + v * kChunkBytes + j * 8192, op.img + chunk_at(op, k0 / kTileM, v, kb) + row_off, 8192, bar);
      }
    }
  }
}

// C[m, n] (+)= sum_k A(m, k) B(n, k) over m < M, n < Nn, K steps [z kps, min(nks, (z + 1) kps)) with z = this CTA's slice.
// part == nullptr: C row-major with leading dimension ldc, accumulate = add to what C holds.  Otherwise slice z writes its own
// [M x Nn] block part + z M Nn (the caller adds the blocks in order).  Block order: n tile fastest, then m tile, then slice.
template <int MNA, int MNB>
__global__ void __launch_bounds__(kThreads, 1) gemm_kernel(const Operand A, const Operand B, int32_t M, int32_t Nn, int32_t nks,
                                                           int32_t kps, int32_t m_tiles, int32_t n_tiles, float *__restrict__ C,
                                                           int32_t ldc, int accumulate, float *__restrict__ part) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + kOffBar;
  auto full = [&](int i) { return bar0 + 8u * i; };
  auto empty = [&](int i) { return bar0 + 8u * (kStages + i); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = (int)(blockIdx.x % (unsigned)n_tiles);
  const int rest = (int)(blockIdx.x / (unsigned)n_tiles);
  const int mt = rest % m_tiles, z = rest / m_tiles;
  const int m0 = mt * kBM, n0 = nt * kBN;
  const int ks0 = z * kps;
  const int steps = min(nks, ks0 + kps) - ks0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(full(i), 1); mbar_init(empty(i), kConsumerWarps); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===== producer: per K step the A and B hi / lo of this tile =====
    if (elect_one()) {
      const uint32_t bytes = operand_bytes<MNA>(A, m0) + operand_bytes<MNB>(B, n0);
      for (int i = 0; i < steps; ++i) {
        const int s = i % kStages, use = i / kStages;
        if (use > 0) mbar_wait_bounded(empty(s), (use - 1) & 1);
        mbar_arrive_expect_tx(full(s), bytes);
        const uint32_t st = sbase + s * kStageBytes;
        copy_operand<MNA>(A, m0, ks0 + i, st, full(s));
        copy_operand<MNB>(B, n0, ks0 + i, st + kOpBytes, full(s));
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of the tile =====
  const int wg = warp >> 2;
  float acc[64], sum[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = sum[i] = 0.f;
  for (int i = 0; i < steps; ++i) {
    const int s = i % kStages;
    mbar_wait_bounded(full(s), (i / kStages) & 1);
    const uint32_t a0 = sbase + s * kStageBytes + wg * 8192;      // this warpgroup's 64 rows (K-major) / 64 columns (MN-major)
    const uint32_t b0 = sbase + s * kStageBytes + kOpBytes;
    wgmma_fence();
#pragma unroll
    for (int k16 = 0; k16 < kBK / 16; ++k16) {
      const uint32_t ao = MNA ? k16 * 2048u : k16 * 32u;      // MN-major: 16 K rows = two 8-row groups; K-major: 16 bf16
      const uint32_t bo = MNB ? k16 * 2048u : k16 * 32u;
      constexpr uint32_t lbo_a = MNA ? 8192u : 16u, lbo_b = MNB ? 8192u : 16u;   // MN-major: the next 64 columns are 8 KB on
      const uint64_t a_hi = gmma_desc(a0 + ao, lbo_a), a_lo = gmma_desc(a0 + kChunkBytes + ao, lbo_a);
      const uint64_t b_hi = gmma_desc(b0 + bo, lbo_b), b_lo = gmma_desc(b0 + kChunkBytes + bo, lbo_b);
      wgmma_n128<MNA, MNB>(acc, a_hi, b_hi, k16 == 0 ? 0u : 1u);
      wgmma_n128<MNA, MNB>(acc, a_hi, b_lo, 1u);
      wgmma_n128<MNA, MNB>(acc, a_lo, b_hi, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty(s));
#pragma unroll
    for (int j = 0; j < 64; ++j) sum[j] += acc[j];
  }

  // epilogue: thread holds rows row0, row0 + 8 and columns 8 j + c2, 8 j + c2 + 1 (j < 16) of its warpgroup's [64 x 128] block
  const int row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c2 = 2 * (lane & 3);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int m = row0 + 8 * hh;
    if (m >= M) continue;
    float *crow = part ? part + ((size_t)z * M + m) * Nn : C + (size_t)m * ldc;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = n0 + 8 * j + c2;
      if (n >= Nn) continue;       // Nn is even: both columns of the pair are valid or neither
      float2 v = make_float2(sum[4 * j + 2 * hh], sum[4 * j + 2 * hh + 1]);
      if (accumulate && !part) {
        const float2 o = *reinterpret_cast<const float2 *>(crow + n);
        v.x += o.x;
        v.y += o.y;
      }
      *reinterpret_cast<float2 *>(crow + n) = v;
    }
  }
}

// C[i] += sum over z of part[z][i], z in order (C dense)
__global__ void __launch_bounds__(256) slices_add_kernel(const float *__restrict__ part, int nz, int64_t count, float *__restrict__ C) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  float s = 0.f;
  for (int z = 0; z < nz; ++z) s += part[(size_t)z * count + i];
  C[i] += s;
}

}  // namespace tcw

namespace {

inline size_t align1k(size_t x) { return (x + 1023) & ~(size_t)1023; }

// Split of the weight-gradient GEMM (K = nodes) over the SMs: the number of slices s <= 32 whose CTAs (tiles x s) fill their
// last wave best, the smallest such s on a tie; then at most one slice per 64-node step.
int tcw_wgrad_split(int32_t N, int32_t D) {
  const int tiles = ((3 * D + tcw::kBM - 1) / tcw::kBM) * ((D + tcw::kBN - 1) / tcw::kBN);
  const int nks = (N + tcw::kBK - 1) / tcw::kBK;
  int best = 1;
  long best_num = 0, best_den = 1;      // fill = tiles s / (waves x SMs), compared as fractions
  for (int s = 1; s <= 32; ++s) {
    const long ctas = (long)tiles * s, waves = (ctas + kNumSMs - 1) / kNumSMs;
    if (ctas * best_den > best_num * waves * kNumSMs) { best = s; best_num = ctas; best_den = waves * kNumSMs; }
  }
  return best < nks ? best : (nks > 0 ? nks : 1);
}
// the split's slices: kps K steps each, the last one kps or fewer
void tcw_slices(int32_t N, int32_t D, int *kps, int *nz) {
  const int nks = (N + tcw::kBK - 1) / tcw::kBK;
  const int split = tcw_wgrad_split(N, D);
  *kps = (nks + split - 1) / split;
  if (*kps < 1) *kps = 1;
  *nz = nks > 0 ? (nks + *kps - 1) / *kps : 1;
}

template <int MNA, int MNB>
int tcw_gemm(tcw::Operand A, tcw::Operand B, int32_t M, int32_t Nn, int32_t K, float *C, int32_t ldc, int accumulate, float *part,
             int kps, cudaStream_t stream) {
  const int nks = (K + tcw::kBK - 1) / tcw::kBK;
  if (M == 0 || Nn == 0 || nks == 0) return DDFA_OK;
  const int m_tiles = (M + tcw::kBM - 1) / tcw::kBM, n_tiles = (Nn + tcw::kBN - 1) / tcw::kBN;
  if (kps <= 0) kps = nks;
  const int nz = (nks + kps - 1) / kps;
  const long long ctas = (long long)m_tiles * n_tiles * nz;
  if (ctas > 0x7fffffffLL) {
    set_error("tensor-core engine (wide): %lld CTAs exceed the grid", ctas);
    return DDFA_ERR_UNSUPPORTED;
  }
  DDFA_CUDA(cudaFuncSetAttribute(tcw::gemm_kernel<MNA, MNB>, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::kSmemAlloc));
  tcw::gemm_kernel<MNA, MNB><<<(unsigned)ctas, tcw::kThreads, tcw::kSmemAlloc, stream>>>(A, B, M, Nn, nks, kps, m_tiles, n_tiles, C, ldc,
                                                                                        accumulate, part);
  DDFA_CHECK_LAUNCH("tcw::gemm_kernel");
  return DDFA_OK;
}

struct FwdScratch {
  uint8_t *s_img, *h_img;
};
FwdScratch fwd_scratch(void *scratch, int32_t N, int32_t D) {
  uint8_t *p = static_cast<uint8_t *>(scratch);
  const size_t img = align1k(tcc::image_bytes_w(N, D));
  return {p, p + img};
}
struct BwdScratch {
  uint8_t *dgi_img, *dgh_img, *s_img, *h_img;
  float *part;
};
BwdScratch bwd_scratch(void *scratch, int32_t N, int32_t D) {
  uint8_t *p = static_cast<uint8_t *>(scratch);
  const size_t q = align1k(tcc::image_bytes_w(N, 3 * D)), a = align1k(tcc::image_bytes_w(N, D));
  return {p, p + q, p + 2 * q, p + 2 * q + a, reinterpret_cast<float *>(p + 2 * q + 2 * a)};
}
const uint8_t *wf_image(const void *weights) { return static_cast<const uint8_t *>(weights); }
const uint8_t *whh_image(const void *weights, int32_t D) {
  return static_cast<const uint8_t *>(weights) + align1k(tcc::image_bytes_w(3 * D, D));
}

}  // namespace

bool gru_tcw_width(int32_t D) { return D >= 192 && D <= 512 && D % 64 == 0; }

size_t gru_tcw_weights_bytes(int32_t D) { return 2 * align1k(tcc::image_bytes_w(3 * D, D)); }

size_t gru_tcw_fwd_scratch_bytes(int32_t N, int32_t D) { return 2 * align1k(tcc::image_bytes_w(N, D)); }

size_t gru_tcw_bwd_scratch_bytes(int32_t N, int32_t D) {
  int kps, nz;
  tcw_slices(N, D, &kps, &nz);
  return 2 * align1k(tcc::image_bytes_w(N, 3 * D)) + 2 * align1k(tcc::image_bytes_w(N, D)) + (size_t)nz * 3 * D * D * sizeof(float);
}

int gru_tcw_prepare(const float *w_fold, const float *w_hh, int32_t D, void *weights, cudaStream_t stream) {
  uint8_t *w = static_cast<uint8_t *>(weights);
  int rc = act_to_image(w_fold, 3 * D, D, w, stream);
  if (rc) return rc;
  return act_to_image(w_hh, 3 * D, D, w + align1k(tcc::image_bytes_w(3 * D, D)), stream);
}

int gru_tcw_fwd_gemms(const float *s, const float *h, int32_t N, int32_t D, const void *weights, void *scratch, float *gi, float *gh,
                      cudaStream_t stream) {
  const FwdScratch w = fwd_scratch(scratch, N, D);
  int rc = act_to_image(s, N, D, w.s_img, stream);
  if (rc) return rc;
  rc = act_to_image(h, N, D, w.h_img, stream);
  if (rc) return rc;
  rc = tcw_gemm<0, 0>({w.s_img, D}, {wf_image(weights), D}, N, 3 * D, D, gi, 3 * D, 0, nullptr, 0, stream);
  if (rc) return rc;
  return tcw_gemm<0, 0>({w.h_img, D}, {whh_image(weights, D), D}, N, 3 * D, D, gh, 3 * D, 0, nullptr, 0, stream);
}

int gru_tcw_bwd_gemms(const float *dgi, const float *dgh, const float *s, const float *h, int32_t N, int32_t D, const void *weights,
                      void *scratch, float *ds, float *dh, float *dw_fold, float *dw_hh, cudaStream_t stream) {
  const BwdScratch w = bwd_scratch(scratch, N, D);
  int rc;
  if ((rc = act_to_image(dgi, N, 3 * D, w.dgi_img, stream))) return rc;
  if ((rc = act_to_image(dgh, N, 3 * D, w.dgh_img, stream))) return rc;
  if ((rc = act_to_image(s, N, D, w.s_img, stream))) return rc;
  if ((rc = act_to_image(h, N, D, w.h_img, stream))) return rc;
  // ds = dgi W' ; dh = dh' z + dgh Whh
  if ((rc = tcw_gemm<0, 1>({w.dgi_img, 3 * D}, {wf_image(weights), D}, N, D, 3 * D, ds, D, 0, nullptr, 0, stream))) return rc;
  if ((rc = tcw_gemm<0, 1>({w.dgh_img, 3 * D}, {whh_image(weights, D), D}, N, D, 3 * D, dh, D, 1, nullptr, 0, stream))) return rc;
  // dw_fold += dgi^T s ; dw_hh += dgh^T h   (K = nodes, split over the SMs, slices added in order)
  int kps, nz;
  tcw_slices(N, D, &kps, &nz);
  const int64_t count = (int64_t)3 * D * D;
  const unsigned add_blocks = (unsigned)((count + 255) / 256);
  if ((rc = tcw_gemm<1, 1>({w.dgi_img, 3 * D}, {w.s_img, D}, 3 * D, D, N, nullptr, D, 0, w.part, kps, stream))) return rc;
  tcw::slices_add_kernel<<<add_blocks, 256, 0, stream>>>(w.part, nz, count, dw_fold);
  DDFA_CHECK_LAUNCH("tcw::slices_add_kernel");
  if ((rc = tcw_gemm<1, 1>({w.dgh_img, 3 * D}, {w.h_img, D}, 3 * D, D, N, nullptr, D, 0, w.part, kps, stream))) return rc;
  tcw::slices_add_kernel<<<add_blocks, 256, 0, stream>>>(w.part, nz, count, dw_hh);
  DDFA_CHECK_LAUNCH("tcw::slices_add_kernel");
  return DDFA_OK;
}

}  // namespace ddfa

extern "C" {

size_t ddfa_gru_tc_wide_gemm_workspace_bytes(int call, int32_t N, int32_t D) {
  using namespace ddfa;
  if (N < 0 || !gru_tcw_width(D) || call < 0 || call > 3) return 0;
  return gru_tcw_weights_bytes(D) + gru_tcw_bwd_scratch_bytes(N, D);
}

int ddfa_gru_tc_wide_gemm(int call, const float *a, const float *b, int32_t N, int32_t D, float *c, void *workspace,
                          size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(call >= 0 && call <= 3, "ddfa_gru_tc_wide_gemm: call must be 0..3 (got %d)", call);
  if (N < 0 || !gru_tcw_width(D)) {
    set_error("ddfa_gru_tc_wide_gemm: the wide tensor-core GEMMs run D = 192 .. 512, D %% 64 == 0 (N=%d D=%d)", N, D);
    return DDFA_ERR_UNSUPPORTED;
  }
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(a && b && c, "ddfa_gru_tc_wide_gemm: NULL pointer");
  // the operands are read with 16-byte loads (to_image_kernel), c is written with 8-byte stores
  DDFA_REQUIRE(aligned16(a) && aligned16(b) && (reinterpret_cast<uintptr_t>(c) & 7) == 0,
               "ddfa_gru_tc_wide_gemm: a and b must be 16-byte aligned, c 8-byte aligned");
  const size_t need = ddfa_gru_tc_wide_gemm_workspace_bytes(call, N, D);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("ddfa_gru_tc_wide_gemm: workspace too small (%zu < %zu)", workspace_bytes, need);
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t stream = as_stream(stream_);
  uint8_t *wimg = static_cast<uint8_t *>(workspace);
  const BwdScratch w = bwd_scratch(wimg + gru_tcw_weights_bytes(D), N, D);
  int rc;
  if (call == 3) {      // c[3D, D] += a[N, 3D]^T b[N, D]
    if ((rc = act_to_image(a, N, 3 * D, w.dgi_img, stream))) return rc;
    if ((rc = act_to_image(b, N, D, w.s_img, stream))) return rc;
    int kps, nz;
    tcw_slices(N, D, &kps, &nz);
    if ((rc = tcw_gemm<1, 1>({w.dgi_img, 3 * D}, {w.s_img, D}, 3 * D, D, N, nullptr, D, 0, w.part, kps, stream))) return rc;
    const int64_t count = (int64_t)3 * D * D;
    tcw::slices_add_kernel<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(w.part, nz, count, c);
    DDFA_CHECK_LAUNCH("tcw::slices_add_kernel");
    return DDFA_OK;
  }
  if ((rc = act_to_image(b, 3 * D, D, wimg, stream))) return rc;      // b = W' or Whh [3D, D], as gru_tcw_prepare packs it
  if (call == 0) {      // c[N, 3D] = a[N, D] b^T
    if ((rc = act_to_image(a, N, D, w.s_img, stream))) return rc;
    return tcw_gemm<0, 0>({w.s_img, D}, {wimg, D}, N, 3 * D, D, c, 3 * D, 0, nullptr, 0, stream);
  }
  // call 1: c[N, D] = a[N, 3D] b ; call 2: c += a b
  if ((rc = act_to_image(a, N, 3 * D, w.dgi_img, stream))) return rc;
  return tcw_gemm<0, 1>({w.dgi_img, 3 * D}, {wimg, D}, N, D, 3 * D, c, D, call == 2, nullptr, 0, stream);
}

size_t ddfa_gru_tc_wide_wgrad_slices(int32_t N, int32_t D) {
  using namespace ddfa;
  if (N < 0 || !gru_tcw_width(D)) return 0;
  int kps, nz;
  tcw_slices(N, D, &kps, &nz);
  return (size_t)nz;
}

}  // extern "C"
