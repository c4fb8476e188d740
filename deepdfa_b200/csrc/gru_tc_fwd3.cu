// Tensor-core engine, forward GRU step (D == 128) on Hopper warpgroup MMA (wgmma), activations streamed as the A operand.
//
// Replaces DGL GatedGraphConv's per-step `a = W h (summed over in-edges); h = GRUCell(a, h)` (reference:
// DDFA/code_gnn/models/flow_gnn/ggnn.py:60-63 -> dgl.nn.GatedGraphConv.forward -> torch.nn.GRUCell) for one step, given
// the edge-gathered sum s = A h and h as activation images:
//     gi = s W'^T + deg * b' + b_ih ,  gh = h Whh^T + b_hh ,  r,z = sigmoid(gi + gh) ,  n = tanh(gi_n + r * gh_n) ,
//     h' = n + z (h - n)
//
// A CTA owns a slice of 32 output columns and streams 128-node tiles:
//   * B = the slice's weights, resident in shared memory for the life of the CTA (96 KB, one bulk copy): for each part
//     (s -> W', h -> Whh) the 96 pre-activation rows [r | z | n] x 32 columns, K = 128, hi and lo bf16, K-major SWIZZLE_128B;
//   * A = the s and h image tiles (K-major SWIZZLE_128B, 128 nodes), two 64 KB stages, one bulk copy per tile;
//   * two consumer warpgroups, 64 nodes each: acc_s = s W'^T over [r | z | gi_n] and acc_h = h Whh^T over [r | z | gh_n]
//     (m64n96k16, bf16x3: x_hi w_hi + x_hi w_lo + x_lo w_hi, fp32 accumulate in registers).  A thread's fragment holds all
//     four pre-activations of its (node, column) pairs, and adjacent column pairs, so the epilogue needs no data exchange.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "tc_common.cuh"

namespace ddfa {
namespace tc3 {
using namespace tcc;

constexpr int kSlices = 4;
constexpr int kSliceCols = kD / kSlices;                  // 32 output columns per CTA
constexpr int kRowsPerPart = 3 * kSliceCols;              // 96 pre-activation rows per part: [r | z | n]
constexpr int kWChunkBytes = kRowsPerPart * 128;          // [96 rows x 64 bf16] = 12 KB
constexpr int kSliceWBytes = 8 * kWChunkBytes;            // [part][hi|lo][kb] = 96 KB
constexpr int kStageBytes = kImageTileBytes;              // 64 KB: one operand tile [hi|lo][kb0|kb1]
constexpr int kOffStage = kSliceWBytes;
constexpr int kOffBias = kOffStage + 2 * kStageBytes;     // 224 KB
constexpr int kBiasSlice = 7 * kSliceCols;                // per slice: const {gi_n, r, z, gh_n} then degree {gi_n, r, z}, 32 columns each
constexpr int kOffBar = kOffBias + kBiasSlice * 4;
constexpr int kSmemAlloc = kOffBar + 5 * 8;               // full[2], empty[2], w_full; the dynamic window is 1024-byte aligned (checked)
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 32;        // two consumer warpgroups + one producer warp
constexpr size_t kPackedWBytes = (size_t)kSlices * kSliceWBytes;   // 384 KB
constexpr size_t kPackedBytes = kPackedWBytes + (size_t)kSlices * kBiasSlice * 4;
static_assert(kSmemAlloc <= 232448, "shared memory budget");

// packed[slice]: chunk (part p, variant v, kb) at ((p * 2 + v) * 2 + kb) * 12 KB; row n = 32 b + c holds
// W_p[b * 128 + 32 slice + c][64 kb .. 64 kb + 63] (W_0 = W', W_1 = Whh; b: 0 r, 1 z, 2 n).  One thread per 8-element unit.
__global__ void pack_kernel(const float *__restrict__ w_fold, const float *__restrict__ w_hh, const float *__restrict__ b_fold,
                            const float *__restrict__ b_ih, const float *__restrict__ b_hh, uint8_t *__restrict__ packed) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= kSlices * 2 * kRowsPerPart * 16) return;
  const int u = idx % 16, n = (idx / 16) % kRowsPerPart, p = (idx / (16 * kRowsPerPart)) % 2, slice = idx / (32 * kRowsPerPart);
  const int kb = u >> 3, k0 = u * 8;
  const float *W = (p == 0 ? w_fold : w_hh) + (size_t)((n / kSliceCols) * kD + slice * kSliceCols + n % kSliceCols) * kD;
  float x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = W[k0 + i];
  uint4 ph, pl;
  split8(x, ph, pl);
  uint8_t *base = packed + (size_t)slice * kSliceWBytes + sw128_offset(n, (u & 7) * 8);
  *reinterpret_cast<uint4 *>(base + ((p * 2 + 0) * 2 + kb) * kWChunkBytes) = ph;
  *reinterpret_cast<uint4 *>(base + ((p * 2 + 1) * 2 + kb) * kWChunkBytes) = pl;
  if (p == 0 && u == 0 && n < kSliceCols) {
    const int t = slice * kSliceCols + n;       // output column
    float *bias = reinterpret_cast<float *>(packed + kPackedWBytes) + slice * kBiasSlice;
    bias[0 * kSliceCols + n] = b_ih[2 * kD + t];
    bias[1 * kSliceCols + n] = b_ih[t] + b_hh[t];
    bias[2 * kSliceCols + n] = b_ih[kD + t] + b_hh[kD + t];
    bias[3 * kSliceCols + n] = b_hh[2 * kD + t];
    bias[4 * kSliceCols + n] = b_fold[2 * kD + t];
    bias[5 * kSliceCols + n] = b_fold[t];
    bias[6 * kSliceCols + n] = b_fold[kD + t];
  }
}

// HIMG: the z*h term reads h from the activation image (h == nullptr) instead of an fp32 plane.
// GATES: 0 = nothing saved (inference), 1 = four fp32 planes (`gates`), 2 = packed 64-bit words (`gates_packed`, pack_gates).
template <bool HIMG, int GATES>
__global__ void __launch_bounds__(kThreads, 1) gru_fwd3_kernel(const uint8_t *__restrict__ s_img, const uint8_t *__restrict__ h_img,
                                                               const float *__restrict__ h, const int32_t *__restrict__ indptr,
                                                               const uint8_t *__restrict__ packed, int32_t N,
                                                               float *__restrict__ h_out, uint8_t *__restrict__ h_out_img,
                                                               float *__restrict__ gates, uint2 *__restrict__ gates_packed, int hints) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  if ((sbase & 1023u) != 0) __trap();        // SWIZZLE_128B operand tiles need 1024-byte alignment
  const uint32_t bar0 = sbase + kOffBar;
  auto full = [&](int i) { return bar0 + 8u * i; };
  auto empty = [&](int i) { return bar0 + 8u * (2 + i); };
  const uint32_t w_full = bar0 + 32u;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slice = blockIdx.x % kSlices;
  const int group = blockIdx.x / kSlices, num_groups = gridDim.x / kSlices;
  const int num_tiles = (N + kTileM - 1) / kTileM;
  const int my_tiles = (num_tiles > group) ? (num_tiles - 1 - group) / num_groups + 1 : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(full(i), 1); mbar_init(empty(i), kConsumerWarps); }
    mbar_init(w_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  const int tron = g_trace_on;
  if (threadIdx.x == 0) trace_stamp(tron, 0, 0);
  pdl_launch_dependents();

  if (warp == kConsumerWarps) {
    // ===== producer: the slice's weights once, then per tile the s tile (stage 0) and the h tile (stage 1) =====
    if (my_tiles > 0 && elect_one()) {
      mbar_arrive_expect_tx(w_full, kSliceWBytes);      // the packed weights are the one input read before pdl_wait (common.cuh)
      bulk_g2s(sbase, packed + (size_t)slice * kSliceWBytes, kSliceWBytes, w_full);
      pdl_wait();      // the images are written by the previous kernels of the chain
      for (int k = 0; k < my_tiles; ++k) {
        const size_t toff = (size_t)(group + k * num_groups) * kImageTileBytes;
        for (int p = 0; p < 2; ++p) {
          if (k > 0) mbar_wait_bounded(empty(p), (k - 1) & 1);
          mbar_arrive_expect_tx(full(p), kStageBytes);
          bulk_g2s(sbase + kOffStage + p * kStageBytes, (p == 0 ? s_img : h_img) + toff, kStageBytes, full(p));
          trace_stamp(tron, k, 1 + p);      // 1: s tile copy issued, 2: h tile copy issued
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns nodes 64 wg .. 64 wg + 63 of every tile =====
  float *sbias = reinterpret_cast<float *>(smem + kOffBias);
  for (int i = threadIdx.x; i < kBiasSlice; i += 32 * kConsumerWarps)
    sbias[i] = __ldcg(reinterpret_cast<const float *>(packed + kPackedWBytes) + slice * kBiasSlice + i);
  asm volatile("bar.sync 1, %0;" ::"n"(32 * kConsumerWarps) : "memory");
  pdl_wait();
  if (my_tiles == 0) return;
  const int wg = warp >> 2;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // fragment rows row0 and row0 + 8 of the tile
  const int c4 = 2 * (lane & 3);                               // fragment columns 8 j + c4, 8 j + c4 + 1
  const size_t plane = (size_t)N * kD;
  const uint64_t pol_gates = l2_policy((hints & 1) ? 1 : 0);      // the saved gates are next read in the backward pass
  const uint64_t pol_next = l2_policy((hints & 16) ? 2 : 0);      // h' and its image feed the next two kernels
  mbar_wait_bounded(w_full, 0);
  const bool tr = (warp == 0 && lane == 0);

  for (int k = 0; k < my_tiles; ++k) {
    const int tile = group + k * num_groups;
    float acc_s[48], acc_h[48];
    if (tr) { trace_stamp(tron, k, 7); trace_stamp(tron, k, 3); }
    mbar_wait_bounded(full(0), k & 1);
    if (tr) trace_stamp(tron, k, 4);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      if (p == 1) {
        mbar_wait_bounded(full(1), k & 1);
        if (tr) trace_stamp(tron, k, 5);
      }
      const uint32_t a0 = sbase + kOffStage + p * kStageBytes + wg * 8192;      // this warpgroup's 64 rows of each chunk
      const uint32_t w0 = sbase + p * 4 * kWChunkBytes;
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          const uint64_t a_hi = gmma_desc(a0 + kb * kChunkBytes + k4 * 32), a_lo = gmma_desc(a0 + (2 + kb) * kChunkBytes + k4 * 32);
          const uint64_t b_hi = gmma_desc(w0 + kb * kWChunkBytes + k4 * 32), b_lo = gmma_desc(w0 + (2 + kb) * kWChunkBytes + k4 * 32);
          const uint32_t acc = (kb == 0 && k4 == 0) ? 0u : 1u;
          if (p == 0) {
            wgmma_n96<0, 0>(acc_s, a_hi, b_hi, acc);
            wgmma_n96<0, 0>(acc_s, a_hi, b_lo, 1u);
            wgmma_n96<0, 0>(acc_s, a_lo, b_hi, 1u);
          } else {
            wgmma_n96<0, 0>(acc_h, a_hi, b_hi, acc);
            wgmma_n96<0, 0>(acc_h, a_hi, b_lo, 1u);
            wgmma_n96<0, 0>(acc_h, a_lo, b_hi, 1u);
          }
        }
      }
      wgmma_commit();
    }
    // operands of the epilogue, requested while the MMAs run: in-degree and h of this thread's 2 rows x 8 columns
    float deg[2], hp[2][8];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t node = (int64_t)tile * kTileM + row0 + 8 * hh;
      const bool valid = node < N;
      deg[hh] = valid ? (float)(__ldcg(indptr + node + 1) - __ldcg(indptr + node)) : 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gcol = slice * kSliceCols + 8 * j + c4;
        if constexpr (HIMG) {      // h = hi + lo of the image (rows past N are zero there)
          const uint32_t whi = __ldcg(reinterpret_cast<const uint32_t *>(h_img + image_offset(node, gcol, 0)));
          const uint32_t wlo = __ldcg(reinterpret_cast<const uint32_t *>(h_img + image_offset(node, gcol, 1)));
          hp[hh][2 * j] = __uint_as_float(whi << 16) + __uint_as_float(wlo << 16);
          hp[hh][2 * j + 1] = __uint_as_float(whi & 0xffff0000u) + __uint_as_float(wlo & 0xffff0000u);
        } else {
          const float2 v = valid ? __ldcg(reinterpret_cast<const float2 *>(h + node * kD + gcol)) : make_float2(0.f, 0.f);
          hp[hh][2 * j] = v.x;
          hp[hh][2 * j + 1] = v.y;
        }
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc_s);
    wgmma_fence_regs(acc_h);
    if (tr) { trace_stamp(tron, k, 6); trace_stamp(tron, k, 8); }
    __syncwarp();
    if (lane == 0) { mbar_arrive(empty(0)); mbar_arrive(empty(1)); }     // this warp's MMAs have read both stages
    if (tr) trace_stamp(tron, k, 9);

#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t node = (int64_t)tile * kTileM + row0 + 8 * hh;
      const bool valid = node < N;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = 8 * j + c4, gcol = slice * kSliceCols + c;
        float hn[2], rr[2], zz[2], nn[2], gg[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 2 * hh + e;
          const float dg = deg[hh];
          const float gin = acc_s[4 * (8 + j) + i] + fmaf(dg, sbias[4 * kSliceCols + c + e], sbias[c + e]);
          const float r = fast_sigmoid(acc_s[4 * j + i] + acc_h[4 * j + i] + fmaf(dg, sbias[5 * kSliceCols + c + e], sbias[kSliceCols + c + e]));
          const float z = fast_sigmoid(acc_s[4 * (4 + j) + i] + acc_h[4 * (4 + j) + i] +
                                       fmaf(dg, sbias[6 * kSliceCols + c + e], sbias[2 * kSliceCols + c + e]));
          const float ghn = acc_h[4 * (8 + j) + i] + sbias[3 * kSliceCols + c + e];
          const float n = fast_tanh(fmaf(r, ghn, gin));
          hn[e] = valid ? fmaf(z, hp[hh][2 * j + e] - n, n) : 0.f;      // rows past N stay zero in the image
          rr[e] = r; zz[e] = z; nn[e] = n; gg[e] = ghn;
        }
        const size_t off = (size_t)node * kD + gcol;
        if (valid && h_out != nullptr) st_f2_hint(h_out + off, make_float2(hn[0], hn[1]), pol_next);
        if constexpr (GATES == 2) {
          if (valid) {
            const uint2 g0 = pack_gates(rr[0], zz[0], nn[0], gg[0]), g1 = pack_gates(rr[1], zz[1], nn[1], gg[1]);
            st_u4_hint(gates_packed + off, make_uint4(g0.x, g0.y, g1.x, g1.y), pol_gates);
          }
        }
        if constexpr (GATES == 1) {
          if (valid) {
            st_f2_hint(gates + off, make_float2(rr[0], rr[1]), pol_gates);
            st_f2_hint(gates + plane + off, make_float2(zz[0], zz[1]), pol_gates);
            st_f2_hint(gates + 2 * plane + off, make_float2(nn[0], nn[1]), pol_gates);
            st_f2_hint(gates + 3 * plane + off, make_float2(gg[0], gg[1]), pol_gates);
          }
        }
        if (h_out_img != nullptr) {      // hi = bf16(x), lo = bf16(x - hi): the values split_bf16 produces
          const uint32_t hw = bf16x2_bits(hn[0], hn[1]);
          const uint32_t lw = bf16x2_bits(hn[0] - __uint_as_float(hw << 16), hn[1] - __uint_as_float(hw & 0xffff0000u));
          st_u32_hint(h_out_img + image_offset(node, gcol, 0), hw, pol_next);
          st_u32_hint(h_out_img + image_offset(node, gcol, 1), lw, pol_next);
        }
      }
    }
    if (tr) trace_stamp(tron, k, 10);
  }
}

}  // namespace tc3

size_t gru_tc3_packed_bytes() { return tc3::kPackedBytes; }

int gru_tc3_prepare(const float *w_fold, const float *b_fold, const float *b_ih, const float *w_hh, const float *b_hh, void *packed,
                    cudaStream_t stream) {
  const int total = tc3::kSlices * 2 * tc3::kRowsPerPart * 16;
  tc3::pack_kernel<<<(total + 127) / 128, 128, 0, stream>>>(w_fold, w_hh, b_fold, b_ih, b_hh, static_cast<uint8_t *>(packed));
  DDFA_CHECK_LAUNCH("tc3::pack_kernel");
  chain_break();
  return DDFA_OK;
}

int gru_tc3_step_fwd(const void *s_img, const void *h_img, const float *h, const int32_t *indptr, int32_t N, float *h_out,
                     void *h_out_img, float *save_gates, void *save_gates_packed, const void *packed, cudaStream_t stream) {
  const int tiles = (N + tcc::kTileM - 1) / tcc::kTileM;
  int groups = kNumSMs / tc3::kSlices;
  if (groups > tiles) groups = tiles;
  if (save_gates && save_gates_packed) {
    set_error("tcgen05 engine (fwd): both gate formats requested");
    return DDFA_ERR_INVALID_ARG;
  }
  if ((h == nullptr && save_gates) ) {
    set_error("tcgen05 engine (fwd): fp32 gate planes go with the fp32 h operand (legacy form)");
    return DDFA_ERR_INVALID_ARG;
  }
  if (tiles == 0) return DDFA_OK;
#define DDFA_FWD3_LAUNCH(HIMG, GATES)                                                                                                     \
  do {                                                                                                                                   \
    DDFA_CUDA(cudaFuncSetAttribute(tc3::gru_fwd3_kernel<HIMG, GATES>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc3::kSmemAlloc));     \
    DDFA_CUDA(launch_chain(2, tc3::gru_fwd3_kernel<HIMG, GATES>, dim3(groups * tc3::kSlices), dim3(tc3::kThreads), tc3::kSmemAlloc,        \
                           stream, static_cast<const uint8_t *>(s_img), static_cast<const uint8_t *>(h_img), h, indptr,                   \
                           static_cast<const uint8_t *>(packed), N, h_out, static_cast<uint8_t *>(h_out_img), save_gates,                \
                           static_cast<uint2 *>(save_gates_packed), l2_hints()));                                                        \
  } while (0)
  if (h) {
    if (save_gates) DDFA_FWD3_LAUNCH(false, 1);
    else if (save_gates_packed) DDFA_FWD3_LAUNCH(false, 2);
    else DDFA_FWD3_LAUNCH(false, 0);
  } else {
    if (save_gates_packed) DDFA_FWD3_LAUNCH(true, 2);
    else DDFA_FWD3_LAUNCH(true, 0);
  }
#undef DDFA_FWD3_LAUNCH
  DDFA_CHECK_LAUNCH("tc3::gru_fwd3_kernel");
  return DDFA_OK;
}

// ---- fp32 [N,D] -> image of D columns (tc_common.cuh: image_offset_w; zero tail rows): h_0 enters the image pipeline here, and
// the wide-width engine (gru_tc_wide.cu) turns its GEMM operands into images with it --------------------------------------------
namespace tc3 {
__global__ void __launch_bounds__(256) to_image_kernel(const float *__restrict__ x, int32_t N, int32_t D, uint8_t *__restrict__ image) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread = 8 consecutive columns of a row
  const int units = D >> 3;
  const int64_t rows = ((int64_t)N + kTileM - 1) / kTileM * kTileM;
  if (t >= rows * units) return;
  const int64_t node = t / units;
  const int col = (int)(t - node * units) * 8;
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (node < N) {
    const float4 a = ldg_nc_f4(x + node * D + col), b = ldg_nc_f4(x + node * D + col + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  uint4 ph, pl;
  split8(v, ph, pl);
  *reinterpret_cast<uint4 *>(image + image_offset_w(node, col, 0, D)) = ph;
  *reinterpret_cast<uint4 *>(image + image_offset_w(node, col, 1, D)) = pl;
}
}  // namespace tc3

size_t act_image_bytes(int64_t n) { return tcc::image_bytes(n); }

int act_to_image(const float *x, int32_t N, int32_t D, void *image, cudaStream_t stream) {
  const int64_t rows = ((int64_t)N + tcc::kTileM - 1) / tcc::kTileM * tcc::kTileM;
  const int64_t total = rows * (D / 8);
  if (total == 0) return DDFA_OK;
  tc3::to_image_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, N, D, static_cast<uint8_t *>(image));
  DDFA_CHECK_LAUNCH("to_image_kernel");
  return DDFA_OK;
}
int act_to_image(const float *x, int32_t N, void *image, cudaStream_t stream) { return act_to_image(x, N, tcc::kD, image, stream); }

// workspace-checked entry points used by gru_step.cu (the forward workspace is exactly the packed weights)
size_t gru_tc2_workspace_bytes() { return gru_tc3_packed_bytes(); }

int gru_tc2_prepare(const float *w_fold, const float *b_fold, const float *b_ih, const float *w_hh, const float *b_hh,
                    void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (workspace == nullptr || workspace_bytes < gru_tc2_workspace_bytes()) {
    set_error("tcgen05 engine: workspace too small (%zu < %zu)", workspace_bytes, gru_tc2_workspace_bytes());
    return DDFA_ERR_WORKSPACE;
  }
  return gru_tc3_prepare(w_fold, b_fold, b_ih, w_hh, b_hh, workspace, stream);
}

int gru_tc2_step_fwd(const void *s_img, const void *h_img, const float *h, const int32_t *indptr, int32_t N, float *h_out,
                     void *h_out_img, float *save_gates, void *save_gates_packed, const void *workspace, size_t workspace_bytes,
                     cudaStream_t stream) {
  if (workspace == nullptr || workspace_bytes < gru_tc2_workspace_bytes()) {
    set_error("tcgen05 engine: workspace too small (%zu < %zu)", workspace_bytes, gru_tc2_workspace_bytes());
    return DDFA_ERR_WORKSPACE;
  }
  return gru_tc3_step_fwd(s_img, h_img, h, indptr, N, h_out, h_out_img, save_gates, save_gates_packed, workspace, stream);
}

int gru_tc3_trace_enable(int on) {
  DDFA_CUDA(cudaMemcpyToSymbol(tcc::g_trace_on, &on, sizeof(int)));
  return DDFA_OK;
}
int gru_tc3_trace_read(void *host, size_t bytes) {
  if (bytes > tcc::kTraceWords * sizeof(long long)) bytes = tcc::kTraceWords * sizeof(long long);
  DDFA_CUDA(cudaMemcpyFromSymbol(host, tcc::g_trace, bytes));
  return DDFA_OK;
}

}  // namespace ddfa
