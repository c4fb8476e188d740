// Tensor-core engine, backward of one GRU step (D == 128) — activation images in, TMA-fed, persistent kernels.
// Backward of the same math the forward kernel implements (gru_tc_fwd3.cu; reference: DDFA/code_gnn/models/flow_gnn/
// ggnn.py:60-63 through dgl.nn.GatedGraphConv / torch.nn.GRUCell autograd).
//
//   (1) gate_bwd_image_kernel   q_r, q_z, q_n, q_nr  <-  (dh', h, r, z, n, gh_n)      elementwise, HBM-bound
//         writes the four q matrices as activation IMAGES, the plane dh' * z (dgrad's elementwise term) and the bias
//         gradients (column sums).  The incoming gradient may be given in two parts, dh' = dh_part + A^T ds_prev: the
//         transposed edge gather of the previous step's ds is folded into this kernel's row loop (no dh' round trip
//         through HBM and one launch less per step).
//   (2) dgrad3_kernel           ds = [q_r q_z q_n] W' ;  dh = dh' * z + [q_r q_z q_nr] Whh      K = 3D
//         wgmma with the q image tiles as the A operand (two 64 KB stages) and 64 columns of the weights resident in shared
//         memory as the B operand; a CTA owns one output (ds or dh) and one column half (see the comment at the kernel)
//   (1+2) bwd_step_fused_kernel  (1) and (2) in one 4-CTA cluster kernel, for the packed saved state (the default path):
//         the gate backward of a tile on TMA-staged operands, the q images handed over through L2, and dh' * z through the
//         rows of dh instead of a plane of its own; (1) then (2) remain the path of the fp32 saved state and the A/B reference
//   (3) wgrad_kernel           dW' += [q_r q_z q_n]^T s ;  dWhh += [q_r q_z q_nr]^T h            K = nodes
//         both operands are read "MN-major" straight from the images (whole 128-node tiles, three 64 KB slots); a CTA keeps
//         one [128 x 128] gate block of the fp32 sum in registers over all its tiles (one wgmma accumulation per tile, added to
//         the running sum with round-to-nearest adds) and writes it to a private global partial
//         at the end; wgrad_reduce_kernel sums the partials once per backward pass.
// Precision: bf16x3 everywhere (hi*hi + hi*lo + lo*hi), fp32 accumulate.
#include <cuda_fp16.h>

#include <atomic>

#include "tc_common.cuh"

namespace ddfa {
namespace tc2b {
using namespace tcc;

constexpr int kThreads = 320, kEpiWarps = 8;

// =================================================================================================
// (1) gate backward -> q images, h image, bias gradients
// =================================================================================================
// Persistent: 2 CTAs per SM, every warp strides over node rows (lane = 4 columns), two rows in flight per warp (12 x 16-byte
// loads outstanding per lane); the seven column sums (bias gradients) stay in registers for the whole kernel and are
// combined once per CTA (r01s ncu: with one CTA per 64 rows the shared/global atomics of that reduction were 22% of the
// kernel and the row loop was load-latency-bound).
constexpr int kGbWarps = 8;
struct GbRow {
  float4 d, hv, rr, zz, nn, gh;
  float deg;
  int tb, te;      // this row's neighbour range in the transposed CSR (fused gather)
};
__device__ __forceinline__ float4 bf16x4_to_f4(const uint2 &p) {
  return make_float4(__uint_as_float(p.x << 16), __uint_as_float(p.x & 0xffff0000u), __uint_as_float(p.y << 16), __uint_as_float(p.y & 0xffff0000u));
}
// Two forms of the saved forward state:
//   fp32:   h = [N,128] plane, gates = four [N,128] planes (r, z, n, gh_n)                       (ddfa_gru_step_bwd_image)
//   packed: h = the activation image the forward GEMM read (hi + lo), gates_packed = [N,128] x 64-bit words (pack_gates)
//           — 64 instead of 96 bytes per lane-row                                               (ddfa_gru_step_bwd_image_v2)
__device__ __forceinline__ void gb_load(GbRow &x, const float *__restrict__ dh_out, const float *__restrict__ h,
                                        const uint8_t *__restrict__ h_img_src, const float *__restrict__ gates,
                                        const uint4 *__restrict__ gates_packed, const int32_t *__restrict__ indptr,
                                        const int32_t *__restrict__ indptr_t, size_t plane, int64_t node, int col, bool ok,
                                        uint64_t pol_saved, uint64_t pol_dh) {
  x.tb = x.te = 0;
  if (ok) {
    if (indptr_t) { x.tb = __ldcg(indptr_t + node); x.te = __ldcg(indptr_t + node + 1); }
    const size_t off = (size_t)node * kD + col;
    x.d = ldg_cg_f4_hint(dh_out + off, pol_dh);
    uint2 hh = make_uint2(0u, 0u), hl = hh;
    uint4 g0 = make_uint4(0u, 0u, 0u, 0u), g1 = g0;
    if (h) x.hv = ldg_cg_f4_hint(h + off, pol_saved);                 // saved activations: last use
    else {
      hh = __ldcg(reinterpret_cast<const uint2 *>(h_img_src + image_offset(node, col, 0)));
      hl = __ldcg(reinterpret_cast<const uint2 *>(h_img_src + image_offset(node, col, 1)));
    }
    if (gates) {
      x.rr = ldg_cg_f4_hint(gates + off, pol_saved);
      x.zz = ldg_cg_f4_hint(gates + plane + off, pol_saved);
      x.nn = ldg_cg_f4_hint(gates + 2 * plane + off, pol_saved);
      x.gh = ldg_cg_f4_hint(gates + 3 * plane + off, pol_saved);
    } else {
      g0 = __ldcg(gates_packed + (off >> 1));          // columns col, col+1: {rz, ng, rz, ng}
      g1 = __ldcg(gates_packed + (off >> 1) + 1);      // columns col+2, col+3
    }
    x.deg = (float)(__ldcg(indptr + node + 1) - __ldcg(indptr + node));
    if (!h) {
      const float4 a = bf16x4_to_f4(hh), b = bf16x4_to_f4(hl);
      x.hv = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    if (!gates) {
      unpack_gates(make_uint2(g0.x, g0.y), x.rr.x, x.zz.x, x.nn.x, x.gh.x);
      unpack_gates(make_uint2(g0.z, g0.w), x.rr.y, x.zz.y, x.nn.y, x.gh.y);
      unpack_gates(make_uint2(g1.x, g1.y), x.rr.z, x.zz.z, x.nn.z, x.gh.z);
      unpack_gates(make_uint2(g1.z, g1.w), x.rr.w, x.zz.w, x.nn.w, x.gh.w);
    }
  }
}

__global__ void __launch_bounds__(32 * kGbWarps, 2) gate_bwd_image_kernel(const float *__restrict__ dh_out, const float *__restrict__ h,
                                                                          const uint8_t *__restrict__ h_img_src,
                                                                          const float *__restrict__ gates, const uint4 *__restrict__ gates_packed,
                                                                          const int32_t *__restrict__ indptr,
                                                                          const float *__restrict__ ds_in, const int32_t *__restrict__ indptr_t,
                                                                          const int32_t *__restrict__ indices_t,
                                                                          int32_t N, uint8_t *__restrict__ q_img, size_t img_stride,
                                                                          uint8_t *__restrict__ h_img, float *__restrict__ dhz,
                                                                          float *__restrict__ db_fold,
                                                                          float *__restrict__ db_ih, float *__restrict__ db_hh, float *__restrict__ bias_slots,
                                                                          int hints) {
  __shared__ float red[kGbWarps][7 * kD];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = lane * 4;
  pdl_launch_dependents();
  pdl_wait();
  const uint64_t pol_saved = l2_policy((hints & 2) ? 1 : 0), pol_tmp = l2_policy((hints & 4) ? 2 : 0), pol_dh = l2_policy((hints & 8) ? 1 : 0);
  const size_t plane = (size_t)N * kD;
  float4 sum[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) sum[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int64_t Npad = ((int64_t)N + kTileM - 1) / kTileM * kTileM;
  const int64_t stride = (int64_t)gridDim.x * kGbWarps;

  auto finish = [&](const GbRow &x, int64_t node, bool ok) {
    float4 qr = make_float4(0.f, 0.f, 0.f, 0.f), qz = qr, qn = qr, qnr = qr, hv = qr;
    if (ok) {
      hv = x.hv;
      st_f4_hint(dhz + (size_t)node * kD + col, make_float4(x.d.x * x.zz.x, x.d.y * x.zz.y, x.d.z * x.zz.z, x.d.w * x.zz.w), pol_tmp);
#define BWDQ(f)                                                      \
  {                                                                  \
    const float dz_ = x.d.f * (x.hv.f - x.nn.f);                     \
    const float dn_ = x.d.f * (1.f - x.zz.f);                        \
    qn.f = dn_ * (1.f - x.nn.f * x.nn.f);                            \
    qz.f = dz_ * x.zz.f * (1.f - x.zz.f);                            \
    qr.f = qn.f * x.gh.f * x.rr.f * (1.f - x.rr.f);                  \
    qnr.f = qn.f * x.rr.f;                                           \
  }
      BWDQ(x) BWDQ(y) BWDQ(z) BWDQ(w)
#undef BWDQ
      f4_add(sum[0], qr); f4_add(sum[1], qz); f4_add(sum[2], qn); f4_add(sum[3], qnr);
      f4_fma(sum[4], x.deg, qr); f4_fma(sum[5], x.deg, qz); f4_fma(sum[6], x.deg, qn);
    }
    // images: rows N..Npad-1 are written as zeros (the weight-gradient GEMM sums over all 128 rows of a tile)
    const size_t o_hi = image_offset(node, col, 0), o_lo = image_offset(node, col, 1);
    uint2 ph, pl;
    split4(qr, ph, pl);  *reinterpret_cast<uint2 *>(q_img + 0 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 0 * img_stride + o_lo) = pl;
    split4(qz, ph, pl);  *reinterpret_cast<uint2 *>(q_img + 1 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 1 * img_stride + o_lo) = pl;
    split4(qn, ph, pl);  *reinterpret_cast<uint2 *>(q_img + 2 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 2 * img_stride + o_lo) = pl;
    split4(qnr, ph, pl); *reinterpret_cast<uint2 *>(q_img + 3 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 3 * img_stride + o_lo) = pl;
    if (h_img) {   // only when the caller did not keep the forward pass's image of h_t
      split4(hv, ph, pl); *reinterpret_cast<uint2 *>(h_img + o_hi) = ph; *reinterpret_cast<uint2 *>(h_img + o_lo) = pl;
    }
  };

  for (int64_t node = (int64_t)blockIdx.x * kGbWarps + warp; node < Npad; node += 2 * stride) {
    const int64_t node2 = node + stride;
    GbRow a, b;
    const bool ok_a = node < N, ok_b = node2 < N;
    gb_load(a, dh_out, h, h_img_src, gates, gates_packed, indptr, indptr_t, plane, node, col, ok_a, pol_saved, pol_dh);
    gb_load(b, dh_out, h, h_img_src, gates, gates_packed, indptr, indptr_t, plane, node2, col, ok_b, pol_saved, pol_dh);
    if (indptr_t) {
      // dh' += sum over the transposed-graph neighbours of ds_in: first up to 4 neighbour ids of both rows, then their
      // rows, all loads of a phase in flight together; longer lists finish in a plain loop (deterministic order)
      int ia[4], ib[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        ia[k] = (a.tb + k < a.te) ? __ldcg(indices_t + a.tb + k) : -1;
        ib[k] = (b.tb + k < b.te) ? __ldcg(indices_t + b.tb + k) : -1;
      }
      float4 va[4], vb[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        va[k] = ia[k] >= 0 ? ldg_cg_f4(ds_in + (size_t)ia[k] * kD + col) : make_float4(0.f, 0.f, 0.f, 0.f);
        vb[k] = ib[k] >= 0 ? ldg_cg_f4(ds_in + (size_t)ib[k] * kD + col) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) { f4_add(a.d, va[k]); f4_add(b.d, vb[k]); }
      for (int j = a.tb + 4; j < a.te; ++j) f4_add(a.d, ldg_cg_f4(ds_in + (size_t)__ldcg(indices_t + j) * kD + col));
      for (int j = b.tb + 4; j < b.te; ++j) f4_add(b.d, ldg_cg_f4(ds_in + (size_t)__ldcg(indices_t + j) * kD + col));
    }
    finish(a, node, ok_a);
    if (node2 < Npad) finish(b, node2, ok_b);
  }
#pragma unroll
  for (int i = 0; i < 7; ++i) *reinterpret_cast<float4 *>(&red[warp][i * kD + col]) = sum[i];
  __syncthreads();
  for (int i = threadIdx.x; i < 7 * kD; i += 32 * kGbWarps) {
    float v_ = 0.f;
#pragma unroll
    for (int w = 0; w < kGbWarps; ++w) v_ += red[w][i];
    if (bias_slots) { bias_slots[(size_t)blockIdx.x * 7 * kD + i] = v_; continue; }      // deterministic mode: bias_slots_reduce_kernel
    const int which = i >> 7, c_ = i & 127;
    // 0:S(q_r) 1:S(q_z) 2:S(q_n) 3:S(q_nr) 4:S(deg q_r) 5:S(deg q_z) 6:S(deg q_n)
    if (which == 0) { atomicAdd(db_ih + c_, v_); atomicAdd(db_hh + c_, v_); }
    else if (which == 1) { atomicAdd(db_ih + kD + c_, v_); atomicAdd(db_hh + kD + c_, v_); }
    else if (which == 2) atomicAdd(db_ih + 2 * kD + c_, v_);
    else if (which == 3) atomicAdd(db_hh + 2 * kD + c_, v_);
    else atomicAdd(db_fold + (which - 4) * kD + c_, v_);
  }
}

// =================================================================================================
// (2) dgrad
// =================================================================================================
//   D[node, col] = Q[node, K] * W[K, col]   (role 0: ds, Q = [q_r q_z q_n], W = W' ; role 1: dh, Q = [q_r q_z q_nr], W = Whh)
//   * B = the CTA's 64 output columns of W, resident in shared memory (K = 384 x 64 columns, hi and lo: 96 KB, one bulk copy);
//   * A = the q image tiles (K-major SWIZZLE_128B, 128 nodes), streamed through two 64 KB stages, one bulk copy per q matrix;
//   * a CTA = (role, column half); two consumer warpgroups of 64 nodes each, m64n64k16, bf16x3, fp32 accumulate in registers.
//     A stage is released as soon as the MMAs of the next q matrix are issued (wgmma_wait<1>), so the copy of the next operand
//     overlaps the MMAs of the current one.
constexpr int kD3Stages = 2;
constexpr int kD3StageBytes = kImageTileBytes;               // one q-matrix tile: [hi|lo][kb0|kb1], 64 KB
constexpr int kD3WChunkBytes = 64 * 128;                     // [64 columns x 64 bf16 of K]
constexpr int kD3WBytes = 12 * kD3WChunkBytes;               // [g][hi|lo][kb] = 96 KB per (role, column half)
constexpr int kD3OffStage = kD3WBytes;
constexpr int kD3OffBar = kD3OffStage + kD3Stages * kD3StageBytes;   // 224 KB
constexpr int kD3SmemAlloc = kD3OffBar + (2 * kD3Stages + 1) * 8 + 8 + 1024;   // barriers, one trace word; + slack for the 1024-byte round-up below
constexpr int kD3Threads = 32 * kEpiWarps + 32;              // two consumer warpgroups + one producer warp
constexpr size_t kD3PackedBytes = (size_t)4 * kD3WBytes;     // [role][column half] = 384 KB
static_assert(kD3SmemAlloc <= 232448, "shared memory budget");

// packed[role][half]: chunk (g, v, kb) at ((g * 2 + v) * 2 + kb) * 8 KB; row n holds W[128 g + 64 kb .. + 63][64 half + n]
// (W = W' or Whh, both [3D x D] row-major).  One thread per 8-element unit.
__global__ void dgrad3_pack_kernel(const float *__restrict__ w_fold, const float *__restrict__ w_hh, uint8_t *__restrict__ packed) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 4 * 3 * 64 * 16) return;
  const int u = idx % 16, n = (idx / 16) % 64, g = (idx / (16 * 64)) % 3, rh = idx / (16 * 64 * 3);
  const int role = rh >> 1, half = rh & 1, kb = u >> 3;
  const float *W = role == 0 ? w_fold : w_hh;
  float x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = W[(size_t)(g * kD + u * 8 + i) * kD + half * 64 + n];
  uint4 ph, pl;
  split8(x, ph, pl);
  uint8_t *base = packed + (size_t)rh * kD3WBytes + sw128_offset(n, (u & 7) * 8);
  *reinterpret_cast<uint4 *>(base + ((g * 2 + 0) * 2 + kb) * kD3WChunkBytes) = ph;
  *reinterpret_cast<uint4 *>(base + ((g * 2 + 1) * 2 + kb) * kD3WChunkBytes) = pl;
}

__global__ void __launch_bounds__(kD3Threads, 1) dgrad3_kernel(const uint8_t *__restrict__ q_img, size_t img_stride,
                                                               const float *__restrict__ dhz, const uint8_t *__restrict__ packed3,
                                                               int32_t N, float *__restrict__ ds, float *__restrict__ dh, int hints) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + kD3OffBar;
  auto full = [&](int i) { return bar0 + 8u * i; };
  auto empty = [&](int i) { return bar0 + 8u * (kD3Stages + i); };
  const uint32_t w_full = bar0 + 8u * (2 * kD3Stages);
  const int tron = (g_trace_on == 1);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rh = blockIdx.x & 3, role = rh >> 1, half = rh & 1;
  const int group = blockIdx.x >> 2, num_groups = gridDim.x >> 2;
  const int num_tiles = (N + kTileM - 1) / kTileM;
  const int my_tiles = (num_tiles > group) ? (num_tiles - 1 - group) / num_groups + 1 : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kD3Stages; ++i) { mbar_init(full(i), 1); mbar_init(empty(i), kEpiWarps); }
    mbar_init(w_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) trace_stamp(tron, 0, 0);
  pdl_launch_dependents();

  if (warp == kEpiWarps) {
    // ===== producer: the weights once, then per tile the three q matrices of this role, one 64 KB copy each =====
    if (my_tiles > 0 && elect_one()) {
      mbar_arrive_expect_tx(w_full, kD3WBytes);
      bulk_g2s(sbase, packed3 + (size_t)rh * kD3WBytes, kD3WBytes, w_full);
      pdl_wait();      // the q images come from the gate backward kernel, the previous kernel of the chain
      const uint64_t pol_q = l2_policy((hints & 64) ? 1 : 0);
      int cc = 0;
      for (int k = 0; k < my_tiles; ++k) {
        const int tile = num_tiles - 1 - (group + k * num_groups);   // back to front: the q tiles written last are still in L2
        for (int g = 0; g < 3; ++g, ++cc) {
          const int m = g < 2 ? g : (role == 0 ? 2 : 3);      // q_r, q_z, then q_n (ds) or q_nr (dh)
          const int stage = cc % kD3Stages, use = cc / kD3Stages;
          if (use > 0) mbar_wait_bounded(empty(stage), (use - 1) & 1);
          mbar_arrive_expect_tx(full(stage), kD3StageBytes);
          bulk_g2s_hint(sbase + kD3OffStage + stage * kD3StageBytes, q_img + (size_t)m * img_stride + (size_t)tile * kImageTileBytes,
                        kD3StageBytes, full(stage), pol_q);
          if (g != 1) trace_stamp(tron, k, g == 0 ? 1 : 2);      // 1: first / 2: last q copy of the tile issued
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns nodes 64 wg .. 64 wg + 63 of every tile =====
  pdl_wait();
  if (my_tiles == 0) return;
  const int wg = warp >> 2;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int col0 = half * 64 + 2 * (lane & 3);
  float *out = role == 0 ? ds : dh;
  const uint64_t pol_tmp = l2_policy((hints & 4) ? 2 : 0);       // ds / dh die after the next kernel has read them
  const uint64_t pol_dhz = l2_policy((hints & 8) ? 1 : 0);       // last read of dh'z
  mbar_wait_bounded(w_full, 0);
  const bool tr = (warp == 0 && lane == 0);
  int cc = 0, pending = -1;      // pending: the stage whose MMAs were issued last and not yet waited for
  for (int k = 0; k < my_tiles; ++k) {
    const int tile = num_tiles - 1 - (group + k * num_groups);
    float acc[32];
    if (tr) { trace_stamp(tron, k, 7); trace_stamp(tron, k, 3); }
    for (int g = 0; g < 3; ++g, ++cc) {
      const int stage = cc % kD3Stages, use = cc / kD3Stages;
      mbar_wait_bounded(full(stage), use & 1);
      if (tr && g != 1) trace_stamp(tron, k, g == 0 ? 4 : 5);      // 4: first / 5: last q tile landed
      wgmma_fence();
      const uint32_t a0 = sbase + kD3OffStage + stage * kD3StageBytes + wg * 8192;
      const uint32_t w0 = sbase + g * 4 * kD3WChunkBytes;
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          const uint64_t a_hi = gmma_desc(a0 + kb * kChunkBytes + k4 * 32), a_lo = gmma_desc(a0 + (2 + kb) * kChunkBytes + k4 * 32);
          const uint64_t b_hi = gmma_desc(w0 + kb * kD3WChunkBytes + k4 * 32), b_lo = gmma_desc(w0 + (2 + kb) * kD3WChunkBytes + k4 * 32);
          wgmma_n64<0, 0>(acc, a_hi, b_hi, (g == 0 && kb == 0 && k4 == 0) ? 0u : 1u);
          wgmma_n64<0, 0>(acc, a_hi, b_lo, 1u);
          wgmma_n64<0, 0>(acc, a_lo, b_hi, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      __syncwarp();
      if (pending >= 0 && lane == 0) mbar_arrive(empty(pending));
      pending = stage;
    }
    // dh = acc + (dh' * z): fetch the elementwise term (written by the gate backward) while the last MMAs run
    float2 dv[2][8];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t node = (int64_t)tile * kTileM + row0 + 8 * hh;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dv[hh][j] = make_float2(0.f, 0.f);
        if (role == 1 && node < N) {
          const float *p = dhz + node * kD + col0 + 8 * j;
          dv[hh][j] = make_float2(ldg_cg_f32_hint(p, pol_dhz), ldg_cg_f32_hint(p + 1, pol_dhz));
        }
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (tr) { trace_stamp(tron, k, 6); trace_stamp(tron, k, 8); }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty(pending));
    pending = -1;
    if (tr) trace_stamp(tron, k, 9);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t node = (int64_t)tile * kTileM + row0 + 8 * hh;
      if (node < N) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          st_f2_hint(out + node * kD + col0 + 8 * j, make_float2(acc[4 * j + 2 * hh] + dv[hh][j].x, acc[4 * j + 2 * hh + 1] + dv[hh][j].y), pol_tmp);
      }
    }
    if (tr) trace_stamp(tron, k, 10);
  }
}

// =================================================================================================
// (1+2) gate backward fused into dgrad: one kernel per backward step (packed saved state)
// =================================================================================================
// No single CTA can both compute q for a tile and run all of dgrad on it: the dgrad CTA of one (role, column half) keeps 96 KB
// of weights resident, and both roles take 384 KB.  So the four dgrad CTAs of a 128-node tile form a thread-block cluster:
//   phase A  CTA rank c (= its (role, half), as in dgrad3_kernel) runs the gate backward on rows 32 c .. 32 c + 31 of the tile:
//            dh', the packed gates and h (image pieces, or fp32 rows at step 0) arrive by TMA bulk copies in one 64 KB stage;
//            the transposed edge gather of ds_in is folded in (register loads, data-dependent addresses).  It writes the four q
//            images (global: the weight-gradient GEMM reads them later; rows N .. Npad-1 as zeros) and dh' * z into the rows
//            of the dh OUTPUT, onto which the dh-role CTAs add acc in phase B — dh' * z never needs a plane of its own (so dh
//            must alias neither dh_out nor ds_in: other clusters are still in phase A when this one writes dh);
//   handover every writer fences its generic-proxy stores against the async proxy (the q tiles are read back by TMA, dh' * z
//            is added to by bulk reductions), then the cluster barrier (arrive.release / wait.acquire);
//   phase B  dgrad3_kernel's MMA loop, unchanged: the three q tiles of the role by bulk copy (L2 hits: written microseconds
//            earlier), m64n64k16 bf16x3, the same MMA order.  The accumulator leaves through shared memory: ds by tensor-map
//            stores, dh by tensor-map fp32 add-reductions onto dh' * z (one rounding to nearest, as the register add of the
//            two-kernel path), so ds and dh are bit-identical to the two-kernel path.
// The phase-A operands of a tile and the q tiles share the two 64 KB stages as one ring, four uses per tile (A, q0, q1, q2):
// the next tile's phase-A copy goes into the stage that q1 releases, so it streams from HBM while phase B runs.  q2's stage
// then holds the staged output until the end of the next tile's phase A, while its copies drain.
// Persistent over tiles, one cluster per 4 SMs; every CTA of a cluster runs the same tiles (each iteration holds a cluster
// barrier).  HF32: h as fp32 rows (step 0: h_0 = x) or the activation image.  CSRP: the CSR scalars / first neighbour ids of the
// folded gather pipelined across tiles, one value per lane (DDFA_TUNE_GATE_BWD_TMA = 2, default; 1 = fetched inside the tile).
constexpr int kGtRows = 32;                                                                            // phase-A rows per CTA
constexpr int kGtOffD = 0, kGtOffG = kGtRows * kD * 4, kGtOffH = kGtOffG + kGtRows * kD * 8;          // 16 KB | 32 KB | 16 KB
static_assert(kGtOffH + kGtRows * kD * 4 == kD3StageBytes, "phase A's operands fill exactly one stage");
static_assert(4 * kGtRows == kTileM, "four CTAs per tile");
constexpr int kGtPre = 2;           // neighbour rows of the folded gather requested ahead of the stage wait, per row
constexpr int kGtRowsPerWarp = kGtRows / kEpiWarps;

__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_n(uint32_t bar, uint32_t n) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(n) : "memory");
}
// Tensor-map copies of one box shared -> global, tracked per issuing thread in bulk groups: a plain store, and one that adds the
// fp32 values onto the destination at L2 (round to nearest even, subnormals kept: the bits of an fp32 register add; DESIGN §3).
// Box rows past the map's row count are not written.
__device__ __forceinline__ void tma_store_2d_hint(const CUtensorMap *tm, uint32_t src, int32_t x, int32_t y, uint64_t pol) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%1, %2}], [%3], %4;" ::"l"(tm), "r"(x), "r"(y),
               "r"(src), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d_hint(const CUtensorMap *tm, uint32_t src, int32_t x, int32_t y, uint64_t pol) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group.L2::cache_hint [%0, {%1, %2}], [%3], %4;" ::"l"(tm),
               "r"(x), "r"(y), "r"(src), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }   // sources read
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }             // writes done

// Phase B's output goes out through the stage that held q2 (always stage 1: four ring uses per tile over two stages).  Warpgroup
// wg's [64 rows x 64 fp32] is two boxes of [64 rows x 32 fp32] in the SWIZZLE_128B layout of the ds / dh tensor maps: row r at
// r x 128 bytes, its 16-byte unit u at (u ^ (r & 7)) x 16.  Box b lies at b x 16 KB + wg x 8 KB, 1024-byte aligned and inside the
// bytes of q2 that wg's own MMAs read (rows 64 wg .. 64 wg + 63 of chunk b), so a warpgroup may overwrite them as soon as all of
// its last MMAs have completed.  The 8 rows of one warp's v2 store cover all 8 unit positions twice: 2 wavefronts per 256 bytes.
constexpr int kD3OutStage = 3 % kD3Stages;
static_assert(4 % kD3Stages == 0, "q2 lands in the same stage every tile");
constexpr uint32_t kOutBoxCols = 32, kOutBoxRows = 64;
static_assert(kOutBoxCols * 4 == 128 && kOutBoxRows * 128 == kChunkBytes / 2, "a box is one warpgroup's half of a chunk");
constexpr int kD3OffPhaseAEnd = kD3OffBar + (2 * kD3Stages + 1) * 8;      // trace: SM clock at which the CTA's last warp ended phase A

template <bool HF32, bool CSRP>
__global__ void __launch_bounds__(kD3Threads, 1) bwd_step_fused_kernel(const float *__restrict__ dh_out, const float *__restrict__ h,
                                                                       const uint8_t *__restrict__ h_img_src, const uint2 *__restrict__ gates_packed,
                                                                       const int32_t *__restrict__ indptr, const float *__restrict__ ds_in,
                                                                       const int32_t *__restrict__ indptr_t, const int32_t *__restrict__ indices_t,
                                                                       int32_t N, uint8_t *__restrict__ q_img, size_t img_stride,
                                                                       const uint8_t *__restrict__ packed3, const __grid_constant__ CUtensorMap tm_ds,
                                                                       const __grid_constant__ CUtensorMap tm_dh, float *__restrict__ dh,
                                                                       float *__restrict__ db_fold, float *__restrict__ db_ih, float *__restrict__ db_hh,
                                                                       float *__restrict__ bias_slots, int hints) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + kD3OffBar;
  auto full = [&](int i) { return bar0 + 8u * i; };
  auto empty = [&](int i) { return bar0 + 8u * (kD3Stages + i); };
  const uint32_t w_full = bar0 + 8u * (2 * kD3Stages);
  const int tron = (g_trace_on == 1);
  unsigned long long *phase_a_end = reinterpret_cast<unsigned long long *>(smem + kD3OffPhaseAEnd);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rh = blockIdx.x & 3, role = rh >> 1, half = rh & 1;      // rh = the CTA's rank in its cluster
  const int cluster = blockIdx.x >> 2, num_clusters = gridDim.x >> 2;
  const int num_tiles = (N + kTileM - 1) / kTileM;
  const int my_tiles = (num_tiles > cluster) ? (num_tiles - 1 - cluster) / num_clusters + 1 : 0;
  const int tile0 = num_tiles - 1 - cluster;
  auto tile_of = [&](int k) { return tile0 - k * num_clusters; };      // back to front, as in dgrad3_kernel

  if (threadIdx.x == 0) {
    for (int i = 0; i < kD3Stages; ++i) { mbar_init(full(i), 1); mbar_init(empty(i), kEpiWarps); }
    mbar_init(w_full, 1);
    mbar_fence_init();
    *phase_a_end = 0ull;
  }
  __syncthreads();
  if (threadIdx.x == 0) trace_stamp(tron, 0, 0);
  pdl_launch_dependents();

  if (warp == kEpiWarps) {
    // ===== producer: the weights once; per tile the phase-A operands of the CTA's 32 rows, then (after the handover) the
    // three q tiles of this role.  All 32 lanes run the loop: every thread of the cluster takes part in its barrier. =====
    const uint64_t pol_saved = l2_policy((hints & 2) ? 1 : 0), pol_dh = l2_policy((hints & 8) ? 1 : 0);
    const uint64_t pol_q = l2_policy((hints & 64) ? 1 : 0);
    if (my_tiles > 0 && elect_one()) {
      mbar_arrive_expect_tx(w_full, kD3WBytes);
      bulk_g2s(sbase, packed3 + (size_t)rh * kD3WBytes, kD3WBytes, w_full);
    }
    __syncwarp();
    pdl_wait();      // dh_out and ds_in come from the previous kernel of the chain
    int cc = 0;
    for (int k = 0; k < my_tiles; ++k, cc += 4) {
      const int tile = tile_of(k);
      if (elect_one()) {
        const int stage = cc % kD3Stages, use = cc / kD3Stages;
        if (use > 0) mbar_wait_bounded(empty(stage), (use - 1) & 1);
        const int64_t r0 = (int64_t)tile * kTileM + kGtRows * rh;
        const int valid = (int)max((int64_t)0, min((int64_t)kGtRows, (int64_t)N - r0));      // rows that exist in the [N, ...] arrays
        const uint32_t dst = sbase + kD3OffStage + stage * kD3StageBytes;
        const uint32_t bytes = (uint32_t)valid * (kD * 4 + kD * 8) + (HF32 ? (uint32_t)valid * kD * 4 : (uint32_t)kGtRows * kD * 4);
        mbar_arrive_expect_tx(full(stage), bytes);
        if (valid > 0) {
          bulk_g2s_hint(dst + kGtOffD, dh_out + r0 * kD, (uint32_t)valid * kD * 4, full(stage), pol_dh);
          bulk_g2s_hint(dst + kGtOffG, gates_packed + r0 * kD, (uint32_t)valid * kD * 8, full(stage), pol_saved);
        }
        if (HF32) {
          if (valid > 0) bulk_g2s_hint(dst + kGtOffH, h + r0 * kD, (uint32_t)valid * kD * 4, full(stage), pol_saved);
        } else {      // the 32 rows of each of the four [128 x 64] bf16 chunks: 4 KB pieces (the image is padded to whole tiles)
          const uint8_t *t0 = h_img_src + (size_t)tile * kImageTileBytes + (size_t)(kGtRows * rh) * 128;
#pragma unroll
          for (int ch = 0; ch < 4; ++ch) bulk_g2s_hint(dst + kGtOffH + ch * (kGtRows * 128), t0 + (size_t)ch * kChunkBytes, kGtRows * 128, full(stage), pol_saved);
        }
      }
      __syncwarp();
      cluster_arrive_release();
      cluster_wait_acquire();
      if (elect_one()) {
        fence_proxy_async_global();      // the q tiles the cluster just wrote are read through the async proxy
        for (int g = 0; g < 3; ++g) {
          const int m = g < 2 ? g : (role == 0 ? 2 : 3);      // q_r, q_z, then q_n (ds) or q_nr (dh)
          const int c = cc + 1 + g, stage = c % kD3Stages, use = c / kD3Stages;
          if (use > 0) mbar_wait_bounded(empty(stage), (use - 1) & 1);
          mbar_arrive_expect_tx(full(stage), kD3StageBytes);
          bulk_g2s_hint(sbase + kD3OffStage + stage * kD3StageBytes, q_img + (size_t)m * img_stride + (size_t)tile * kImageTileBytes,
                        kD3StageBytes, full(stage), pol_q);
          if (g != 1) trace_stamp(tron, k, g == 0 ? 1 : 2);      // 1: first / 2: last q copy of the tile issued
        }
      }
      __syncwarp();
    }
  } else {
    // ===== consumers: phase A, warp w owns rows w + 8 j (j < 4) of the CTA's 32; phase B, warpgroup wg owns nodes 64 wg .. + 63 =====
    pdl_wait();
    const int col = lane * 4;
    // L2 policy (created where it is used: 64-bit values live across the whole loop made the kernel spill)
    // pol_tmp: ds / dh / dh' * z die after the next kernel has read them
#define DDFA_POL_TMP l2_policy((hints & 4) ? 2 : 0)
    const int wg = warp >> 2;
    const bool tr = (warp == 0 && lane == 0);
    float4 sum[7];      // the seven column sums (bias gradients) over all the warp's rows, combined once at the end
#pragma unroll
    for (int i = 0; i < 7; ++i) sum[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    // The CSR data of the warp's four rows — indptr (in-degree), indptr_t and the first kGtPre transposed neighbour ids — is a
    // chain of dependent global loads (indptr_t -> indices_t -> ds row), warp-uniform, so with CSRP it is kept ONE VALUE PER LANE
    // and pipelined across tiles: lanes 0-7 hold indptr[node_r + {0,1}], lanes 8-15 indptr_t[node_r + {0,1}] (r = (lane >> 1) & 3)
    // of a tile, lanes 16-23 its ids id[r][q] (q = lane & 1); tile k requests the scalars of tile k + 2 and the ids of tile k + 1
    // and broadcasts its own by shuffle — only the ds rows themselves are requested in the tile that adds them.
    static_assert(kGtPre == 2 && kGtRowsPerWarp == 4, "lane slots below assume four rows per warp and two prefetched neighbours per row");
    auto node_of = [&](int tile, int r) { return (int64_t)tile * kTileM + kGtRows * rh + warp + kEpiWarps * r; };
    auto load_scalars = [&](int kk) -> int {
      int v = 0;
      if (kk < my_tiles && lane < 16) {
        const int64_t nd = node_of(tile_of(kk), (lane >> 1) & 3);
        const int32_t *base = lane < 8 ? indptr : indptr_t;
        if (nd < N && base) v = __ldcg(base + nd + (lane & 1));
      }
      return v;
    };
    auto load_ids = [&](int sc) -> int {
      const int r_ = (lane >> 1) & 3, q_ = lane & 1;
      const int tb_ = __shfl_sync(0xffffffffu, sc, 8 + 2 * r_), te_ = __shfl_sync(0xffffffffu, sc, 9 + 2 * r_);
      int v = -1;
      if (lane >= 16 && lane < 24 && tb_ + q_ < te_) v = __ldcg(indices_t + tb_ + q_);
      return v;
    };
    int sc_cur = 0, sc_next = 0, id_cur = -1;
    if constexpr (CSRP) {
      sc_cur = load_scalars(0); sc_next = load_scalars(1);
      id_cur = load_ids(sc_cur);
    }
    int cc = 0;
    for (int k = 0; k < my_tiles; ++k) {
      const int tile = tile_of(k);
      // ---------------- phase A ----------------
      {
        const int stage = cc % kD3Stages, use = cc / kD3Stages;
        ++cc;
        const int64_t node0 = node_of(tile, 0);      // row r of the warp is node0 + kEpiWarps r
        bool ok[kGtRowsPerWarp];
        int tb[kGtRowsPerWarp], te[kGtRowsPerWarp];
        float deg[kGtRowsPerWarp];
        int id[kGtRowsPerWarp][kGtPre];      // the first kGtPre neighbours of each row (a CFG node has ~2 in-edges); longer lists finish below
        if constexpr (CSRP) {
          const int sc_next2 = load_scalars(k + 2);
          const int id_next = load_ids(sc_next);
#pragma unroll
          for (int r = 0; r < kGtRowsPerWarp; ++r) {
            ok[r] = node0 + kEpiWarps * r < N;
            deg[r] = (float)(__shfl_sync(0xffffffffu, sc_cur, 2 * r + 1) - __shfl_sync(0xffffffffu, sc_cur, 2 * r));
            tb[r] = __shfl_sync(0xffffffffu, sc_cur, 8 + 2 * r); te[r] = __shfl_sync(0xffffffffu, sc_cur, 9 + 2 * r);
#pragma unroll
            for (int q = 0; q < kGtPre; ++q) id[r][q] = __shfl_sync(0xffffffffu, id_cur, 16 + 2 * r + q);
          }
          sc_cur = sc_next; sc_next = sc_next2; id_cur = id_next;
        } else {      // everything requested inside the tile (global, independent of the staged operands: before the wait)
#pragma unroll
          for (int r = 0; r < kGtRowsPerWarp; ++r) {
            const int64_t nd = node0 + kEpiWarps * r;
            ok[r] = nd < N;
            tb[r] = te[r] = 0;
            deg[r] = 0.f;
            if (ok[r]) {
              deg[r] = (float)(__ldcg(indptr + nd + 1) - __ldcg(indptr + nd));
              if (indptr_t) { tb[r] = __ldcg(indptr_t + nd); te[r] = __ldcg(indptr_t + nd + 1); }
            }
          }
#pragma unroll
          for (int r = 0; r < kGtRowsPerWarp; ++r)
#pragma unroll
            for (int q = 0; q < kGtPre; ++q) id[r][q] = (tb[r] + q < te[r]) ? __ldcg(indices_t + tb[r] + q) : -1;
        }
        float4 gv[kGtRowsPerWarp][kGtPre];
#pragma unroll
        for (int r = 0; r < kGtRowsPerWarp; ++r)
#pragma unroll
          for (int q = 0; q < kGtPre; ++q) gv[r][q] = id[r][q] >= 0 ? ldg_cg_f4(ds_in + (size_t)id[r][q] * kD + col) : make_float4(0.f, 0.f, 0.f, 0.f);
        mbar_wait_bounded(full(stage), use & 1);
        const uint8_t *st = smem + kD3OffStage + stage * kD3StageBytes;
#pragma unroll
        for (int r = 0; r < kGtRowsPerWarp; ++r) {
          const int row = warp + kEpiWarps * r;             // row inside the CTA's 32
          float4 d = make_float4(0.f, 0.f, 0.f, 0.f), hv = d, rr = d, zz = d, nn = d, gh = d;
          if (ok[r]) {
            d = *reinterpret_cast<const float4 *>(st + kGtOffD + row * (kD * 4) + col * 4);
            const uint4 g0 = *reinterpret_cast<const uint4 *>(st + kGtOffG + row * (kD * 8) + col * 8);
            const uint4 g1 = *reinterpret_cast<const uint4 *>(st + kGtOffG + row * (kD * 8) + col * 8 + 16);
            unpack_gates(make_uint2(g0.x, g0.y), rr.x, zz.x, nn.x, gh.x);
            unpack_gates(make_uint2(g0.z, g0.w), rr.y, zz.y, nn.y, gh.y);
            unpack_gates(make_uint2(g1.x, g1.y), rr.z, zz.z, nn.z, gh.z);
            unpack_gates(make_uint2(g1.z, g1.w), rr.w, zz.w, nn.w, gh.w);
            if (HF32) {
              hv = *reinterpret_cast<const float4 *>(st + kGtOffH + row * (kD * 4) + col * 4);
            } else {      // piece [v][kb = col / 64] of 32 rows x 128 B; 16-byte units swizzled by (tile row) & 7 == row & 7 (32 rh is a multiple of 8)
              const uint32_t off = (uint32_t)((col >> 6) * (kGtRows * 128) + row * 128 + (((((col & 63) >> 3) ^ (row & 7)) & 7) << 4) + (col & 7) * 2);
              const uint2 hh = *reinterpret_cast<const uint2 *>(st + kGtOffH + off);
              const uint2 hl = *reinterpret_cast<const uint2 *>(st + kGtOffH + 2 * (kGtRows * 128) + off);
              const float4 a = bf16x4_to_f4(hh), b = bf16x4_to_f4(hl);
              hv = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
            }
#pragma unroll
            for (int q = 0; q < kGtPre; ++q) f4_add(d, gv[r][q]);
            for (int j = tb[r] + kGtPre; j < te[r]; ++j) f4_add(d, ldg_cg_f4(ds_in + (size_t)__ldcg(indices_t + j) * kD + col));
          }
          float4 qr = make_float4(0.f, 0.f, 0.f, 0.f), qz = qr, qn = qr, qnr = qr;
          const int64_t node = node0 + kEpiWarps * r;
          if (ok[r]) {
            st_f4_hint(dh + (size_t)node * kD + col, make_float4(d.x * zz.x, d.y * zz.y, d.z * zz.z, d.w * zz.w), DDFA_POL_TMP);
#define BWDQ2(f)                                         \
  {                                                      \
    const float dz_ = d.f * (hv.f - nn.f);               \
    const float dn_ = d.f * (1.f - zz.f);                \
    qn.f = dn_ * (1.f - nn.f * nn.f);                    \
    qz.f = dz_ * zz.f * (1.f - zz.f);                    \
    qr.f = qn.f * gh.f * rr.f * (1.f - rr.f);            \
    qnr.f = qn.f * rr.f;                                 \
  }
            BWDQ2(x) BWDQ2(y) BWDQ2(z) BWDQ2(w)
#undef BWDQ2
            f4_add(sum[0], qr); f4_add(sum[1], qz); f4_add(sum[2], qn); f4_add(sum[3], qnr);
            f4_fma(sum[4], deg[r], qr); f4_fma(sum[5], deg[r], qz); f4_fma(sum[6], deg[r], qn);
          }
          // rows N .. Npad-1 are written as zeros (the weight-gradient GEMM sums over all 128 rows of a tile)
          const size_t o_hi = image_offset(node, col, 0), o_lo = image_offset(node, col, 1);
          uint2 ph, pl;
          split4(qr, ph, pl);  *reinterpret_cast<uint2 *>(q_img + 0 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 0 * img_stride + o_lo) = pl;
          split4(qz, ph, pl);  *reinterpret_cast<uint2 *>(q_img + 1 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 1 * img_stride + o_lo) = pl;
          split4(qn, ph, pl);  *reinterpret_cast<uint2 *>(q_img + 2 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 2 * img_stride + o_lo) = pl;
          split4(qnr, ph, pl); *reinterpret_cast<uint2 *>(q_img + 3 * img_stride + o_hi) = ph; *reinterpret_cast<uint2 *>(q_img + 3 * img_stride + o_lo) = pl;
        }
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(empty(stage));      // this warp has read its rows of the stage
          if (tron) atomicMax(phase_a_end, (unsigned long long)clock64());      // clock64 only grows: no reset between tiles
        }
      }
      // the previous tile's output has been read out of its stage (long ago: its copies drained during this phase A): hand the
      // stage back for this tile's first q copy, which the producer issues only after the handover below — four arrivals per
      // warpgroup, as the MMA loop makes for the other uses
      if (k > 0 && (warp & 3) == 0) {
        bulk_wait_read_all();
        __syncwarp();
        if (lane == 0) mbar_arrive_n(empty(kD3OutStage), kEpiWarps / 2);
      }
      // ---------------- handover: q and dh' * z of the whole tile visible to the cluster ----------------
      fence_proxy_async_global();
      cluster_arrive_release();
      cluster_wait_acquire();
      if (tr) {
        trace_stamp(tron, k, 11);                                   // 11: handover done
        trace_put(tron, k, 14, (long long)*(volatile unsigned long long *)phase_a_end);      // 14: the CTA's last warp ended phase A
      }
      if ((warp & 3) == 0 && role == 1) fence_proxy_async_global();      // dh' * z (generic stores of the cluster) is added to by the async proxy
      // ---------------- phase B: dgrad3_kernel's loop ----------------
      if (k == 0) mbar_wait_bounded(w_full, 0);
      float acc[32];
      int pending = -1;      // the stage whose MMAs were issued last and not yet waited for
      if (tr) { trace_stamp(tron, k, 7); trace_stamp(tron, k, 3); }
      for (int g = 0; g < 3; ++g, ++cc) {
        const int stage = cc % kD3Stages, use = cc / kD3Stages;
        mbar_wait_bounded(full(stage), use & 1);
        if (tr && g != 1) trace_stamp(tron, k, g == 0 ? 4 : 5);      // 4: first / 5: last q tile landed
        wgmma_fence();
        const uint32_t a0 = sbase + kD3OffStage + stage * kD3StageBytes + wg * 8192;
        const uint32_t w0 = sbase + g * 4 * kD3WChunkBytes;
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
          for (int k4 = 0; k4 < 4; ++k4) {
            const uint64_t a_hi = gmma_desc(a0 + kb * kChunkBytes + k4 * 32), a_lo = gmma_desc(a0 + (2 + kb) * kChunkBytes + k4 * 32);
            const uint64_t b_hi = gmma_desc(w0 + kb * kD3WChunkBytes + k4 * 32), b_lo = gmma_desc(w0 + (2 + kb) * kD3WChunkBytes + k4 * 32);
            wgmma_n64<0, 0>(acc, a_hi, b_hi, (g == 0 && kb == 0 && k4 == 0) ? 0u : 1u);
            wgmma_n64<0, 0>(acc, a_hi, b_lo, 1u);
            wgmma_n64<0, 0>(acc, a_lo, b_hi, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        __syncwarp();
        if (pending >= 0 && lane == 0) mbar_arrive(empty(pending));
        pending = stage;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (tr) { trace_stamp(tron, k, 6); trace_stamp(tron, k, 8); trace_stamp(tron, k, 9); }
      // ds = acc; dh = acc + dh' * z, the elementwise term phase A wrote into dh's rows.  The fragment goes into q2's stage as two
      // swizzled boxes per warpgroup (see kOutBoxCols), then one tensor-map copy per box leaves the SM — for dh one that adds onto
      // dh' * z in L2, so the SM never reads it back.  The maps end at row N: ds and dh are unpadded [N, 128] planes.
      const uint32_t st_base = sbase + kD3OffStage + kD3OutStage * kD3StageBytes;      // == pending
      // a warp's wait covers the rows of q2 its own MMAs read (16 per chunk); it stages into rows its siblings read
      if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
      else asm volatile("bar.sync 3, 128;" ::: "memory");
      uint32_t tid;      // re-read here: addresses derived from it and kept across the tile loop made the kernel spill
      asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
      // fragment row (tid >> 5 & 3) x 16 + (tid >> 2 & 7) + 8 hh; its row & 7 is tid >> 2 & 7.  Column 8 j + 2 (tid & 3) + e lies
      // in box j / 4, unit 2 (j % 4) + (tid >> 1 & 1), byte 8 (tid & 1) + 4 e of the unit.
      const uint32_t sw = ((tid >> 1 & 1) ^ (tid >> 2)) & 7;      // the unit's low bit and the row's swizzle, folded
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t rowp = st_base + (tid >> 7) * (kChunkBytes / 2) + ((tid >> 5 & 3) * 16 + (tid >> 2 & 7) + 8 * hh) * 128 + 8 * (tid & 1);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(rowp + (j >> 2) * kChunkBytes + (((2 * (j & 3)) ^ sw) << 4)),
                       "f"(acc[4 * j + 2 * hh]), "f"(acc[4 * j + 2 * hh + 1])
                       : "memory");
      }
      fence_proxy_async_shared();
      if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");      // the warpgroup's 64 rows are staged
      else asm volatile("bar.sync 3, 128;" ::: "memory");
      if ((warp & 3) == 0 && elect_one()) {      // one thread per warpgroup issues its copies (uniform operands: straight-line issue)
        const int32_t y = tile * kTileM + wg * 64;
        if (y < N) {      // the map clips a partial box; a box wholly past N is not issued
          const uint64_t pol_tmp = DDFA_POL_TMP;
          const uint32_t src = st_base + wg * (kChunkBytes / 2);
#pragma unroll
          for (int b = 0; b < 2; ++b) {
            const int32_t x = half * 64 + b * (int)kOutBoxCols;
            if (role == 0) tma_store_2d_hint(&tm_ds, src + b * kChunkBytes, x, y, pol_tmp);
            else tma_reduce_add_2d_hint(&tm_dh, src + b * kChunkBytes, x, y, pol_tmp);
          }
        }
        bulk_commit();
        trace_stamp(tron, k, 12 + wg);      // 12 / 13: warpgroup 0 / 1 has issued its copies
      }
      __syncwarp();
      if (tr) trace_stamp(tron, k, 10);
    }
#undef DDFA_POL_TMP
    bulk_wait_all();      // ds / dh complete before the CTA exits: the next kernels of the step read them
    // bias gradients: the warps' column sums through the stages, once both warpgroups are past their last MMAs
    asm volatile("bar.sync 1, %0;" ::"n"(32 * kEpiWarps) : "memory");
    float *red = reinterpret_cast<float *>(smem + kD3OffStage);
#pragma unroll
    for (int i = 0; i < 7; ++i) *reinterpret_cast<float4 *>(&red[(warp * 7 + i) * kD + col]) = sum[i];
  }
  __syncthreads();
  const float *red = reinterpret_cast<const float *>(smem + kD3OffStage);
  for (int i = threadIdx.x; i < 7 * kD; i += kD3Threads) {
    float v_ = 0.f;
#pragma unroll
    for (int w = 0; w < kEpiWarps; ++w) v_ += red[(w * 7) * kD + i];
    if (bias_slots) { bias_slots[(size_t)blockIdx.x * 7 * kD + i] = v_; continue; }      // deterministic mode: bias_slots_reduce_kernel
    const int which = i >> 7, c_ = i & 127;
    // 0:S(q_r) 1:S(q_z) 2:S(q_n) 3:S(q_nr) 4:S(deg q_r) 5:S(deg q_z) 6:S(deg q_n)
    if (which == 0) { atomicAdd(db_ih + c_, v_); atomicAdd(db_hh + c_, v_); }
    else if (which == 1) { atomicAdd(db_ih + kD + c_, v_); atomicAdd(db_hh + kD + c_, v_); }
    else if (which == 2) atomicAdd(db_ih + 2 * kD + c_, v_);
    else if (which == 3) atomicAdd(db_hh + 2 * kD + c_, v_);
    else atomicAdd(db_fold + (which - 4) * kD + c_, v_);
  }
}

// =================================================================================================
// (3) wgrad
// =================================================================================================
//   dW'[128 g + m, n] += sum_node q_g[node, m] s[node, n] ;  dWhh likewise with h (K = nodes)
// grid = (ctas, 6): blockIdx.y = 3 role + g.  A CTA owns one [128 x 128] gate block of one role: per tile it streams the s / h tile
// (B) and the q_g tile (A) through a ring of three 64 KB slots; both operands are read MN-major straight from the images.  Two
// consumer warpgroups hold rows 0-63 / 64-127 of the block (m64n128k16, bf16x3) in registers over all the CTA's tiles and
// write them to a private partial sum at the end.
// partial: [2][ctas][384*128] fp32, private per CTA: accumulate (first == 0) or overwrite (first != 0); the sum over CTAs
// is taken once per backward pass by wgrad_reduce_kernel (no atomics on the hot path).
// One launch may cover several time steps (K = steps x nodes): the q images of step t are at q_img + t * step_stride, its
// B operands are batch.s_img[t] / batch.h_img[t].  Batching all T steps of a backward pass into one launch removes T-1
// epilogues (read-modify-write of the private partial sums), T-1 pipeline ramps and T-1 launches.
constexpr int kWgSlotBytes = kImageTileBytes;             // 64 KB
constexpr int kWgSlots = 3;
constexpr int kWgOffBar = kWgSlots * kWgSlotBytes;        // 192 KB
constexpr int kWgSmemAlloc = kWgOffBar + 2 * kWgSlots * 8 + 1024;
constexpr int kWgThreads = 32 * kEpiWarps + 32;
constexpr size_t kWgPartialFloats = (size_t)3 * kD * kD;  // one CTA slot's [384 x 128] partial sum
constexpr int kWgMaxSteps = 16;
struct WgBatch {
  const uint8_t *s_img[kWgMaxSteps];
  const uint8_t *h_img[kWgMaxSteps];
  int32_t steps;
};
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const uint8_t *__restrict__ q_img, size_t img_stride, size_t step_stride,
                                                              const __grid_constant__ WgBatch batch,
                                                              int32_t N, float *__restrict__ partial, int first, int hints) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + kWgOffBar;
  auto full = [&](int i) { return bar0 + 8u * i; };
  auto empty = [&](int i) { return bar0 + 8u * (kWgSlots + i); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = blockIdx.y / 3, g = blockIdx.y % 3;
  const int qm = g < 2 ? g : (role == 0 ? 2 : 3);            // q_r, q_z, then q_n (dW') or q_nr (dWhh)
  const int num_tiles = (N + kTileM - 1) / kTileM;           // per time step
  const int all_tiles = num_tiles * batch.steps;
  const int my_tiles = (all_tiles > (int)blockIdx.x) ? (all_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgSlots; ++i) { mbar_init(full(i), 1); mbar_init(empty(i), kEpiWarps); }
    mbar_fence_init();
  }
  __syncthreads();
  const int tron = (g_trace_on == 2) && blockIdx.y == 0;   // timeline of the gate-block-0 CTAs of dW' (ddfa_debug_set key 2, value 2)
  if (threadIdx.x == 0) trace_stamp(tron, 0, 0);

  if (warp == kEpiWarps) {
    // ===== producer: per tile the B tile (s or h) then the A tile (q_g) =====
    if (elect_one()) {
      const uint64_t pol_wg = l2_policy((hints & 32) ? 1 : 0);     // every operand of the batched launch is read once
      for (int i = 0; i < my_tiles; ++i) {
        const int idx = (int)blockIdx.x + i * (int)gridDim.x;
        const int t = idx / num_tiles, tile = idx - t * num_tiles;
        for (int w = 0; w < 2; ++w) {
          const int cc = 2 * i + w, slot = cc % kWgSlots, use = cc / kWgSlots;
          if (use > 0) mbar_wait_bounded(empty(slot), (use - 1) & 1);
          const uint8_t *src = w == 0 ? (role == 0 ? batch.s_img[t] : batch.h_img[t]) : q_img + (size_t)t * step_stride + (size_t)qm * img_stride;
          mbar_arrive_expect_tx(full(slot), kWgSlotBytes);
          bulk_g2s_hint(sbase + slot * kWgSlotBytes, src + (size_t)tile * kImageTileBytes, kWgSlotBytes, full(slot), pol_wg);
          trace_stamp(tron, i, 1 + w);      // 1: B (s / h) copy issued, 2: A (q) copy issued
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  // acc: this tile's wgmma accumulator (restarted every tile); sum: the running sum over the CTA's tiles, in ordinary fp32 adds.
  // Chaining all tiles inside the wgmma accumulator biased the sum toward zero by about 2e-7 per tile (the tensor core's fp32
  // accumulation does not round to nearest): -1e-4 of dW' / dWhh at 447 tiles per CTA (C1, T = 8, tests/test_scale_gpu.py).
  float acc[64], sum[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = sum[i] = 0.f;
  for (int i = 0; i < my_tiles; ++i) {
    const int cb = 2 * i, ca = 2 * i + 1;
    mbar_wait_bounded(full(cb % kWgSlots), (cb / kWgSlots) & 1);
    if (warp == 0 && lane == 0) trace_stamp(tron, i, 3);
    mbar_wait_bounded(full(ca % kWgSlots), (ca / kWgSlots) & 1);
    if (warp == 0 && lane == 0) { trace_stamp(tron, i, 4); trace_stamp(tron, i, 5); }
    const uint32_t b0 = sbase + (cb % kWgSlots) * kWgSlotBytes;
    const uint32_t a0 = sbase + (ca % kWgSlots) * kWgSlotBytes + wg * kChunkBytes;      // q columns 64 wg .. 64 wg + 63
    constexpr uint32_t vs = 2 * kChunkBytes;                                              // hi -> lo variant
    wgmma_fence();
#pragma unroll
    for (int k16 = 0; k16 < kTileM / 16; ++k16) {
      const uint32_t koff = (uint32_t)k16 * 2048u;      // 16 nodes = two 8-node groups of 1024 B
      const uint64_t a_hi = gmma_desc(a0 + koff, kChunkBytes), a_lo = gmma_desc(a0 + vs + koff, kChunkBytes);
      const uint64_t b_hi = gmma_desc(b0 + koff, kChunkBytes), b_lo = gmma_desc(b0 + vs + koff, kChunkBytes);
      wgmma_n128<1, 1>(acc, a_hi, b_hi, k16 == 0 ? 0u : 1u);
      wgmma_n128<1, 1>(acc, a_lo, b_hi, 1u);
      wgmma_n128<1, 1>(acc, a_hi, b_lo, 1u);
    }
    wgmma_commit();
    if (warp == 0 && lane == 0) trace_stamp(tron, i, 6);
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) { mbar_arrive(empty(cb % kWgSlots)); mbar_arrive(empty(ca % kWgSlots)); }
#pragma unroll
    for (int j = 0; j < 64; ++j) sum[j] += acc[j];
  }
  if (warp == 0 && lane == 0) trace_stamp(tron, 0, 8);
  // this CTA's private partial: rows 128 g + (fragment row), 128 columns; every CTA writes its slot (zeros if it owns no tile)
  float *dst = partial + ((size_t)role * gridDim.x + blockIdx.x) * kWgPartialFloats;
  const int row0 = g * kD + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float *rowp = dst + (size_t)(row0 + 8 * hh) * kD + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float2 v = make_float2(sum[4 * j + 2 * hh], sum[4 * j + 2 * hh + 1]);
      if (!first) {
        const float2 o = *reinterpret_cast<const float2 *>(rowp + 8 * j);
        v.x += o.x;
        v.y += o.y;
      }
      *reinterpret_cast<float2 *>(rowp + 8 * j) = v;
    }
  }
  if (warp == 0 && lane == 0) trace_stamp(tron, 0, 10);
}

// dW'[384,128] += sum_cta partial[0][cta] ; dWhh += sum_cta partial[1][cta]     (once per backward pass)
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float *__restrict__ partial, int ctas, float *__restrict__ dw_fold,
                                                           float *__restrict__ dw_hh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;        // float4 index inside one [384 x 128] matrix
  const int role = blockIdx.y;
  if (i >= (int)(kWgPartialFloats / 4)) return;
  const float4 *src = reinterpret_cast<const float4 *>(partial + (size_t)role * ctas * kWgPartialFloats) + i;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < ctas; ++c) f4_add(s, src[(size_t)c * (kWgPartialFloats / 4)]);
  float4 *dst = reinterpret_cast<float4 *>(role == 0 ? dw_fold : dw_hh) + i;
  float4 d = *dst;
  f4_add(d, s);
  *dst = d;
}

// Deterministic mode: the bias-gradient column sums of the step's CTAs (slot c = CTA c, 7 x 128 floats, the order of the epilogues
// above), added in CTA order — one thread per column.
constexpr int kBiasSlots = 2 * kNumSMs;      // the largest grid of the step's first kernel (gate_bwd_image_kernel)
__global__ void __launch_bounds__(128) bias_slots_reduce_kernel(const float *__restrict__ slots, int ctas, float *__restrict__ db_fold,
                                                                float *__restrict__ db_ih, float *__restrict__ db_hh) {
  const int i = blockIdx.x * 128 + threadIdx.x;
  const int which = i >> 7, c_ = i & 127;
  float v_ = 0.f;
  for (int c = 0; c < ctas; ++c) v_ += slots[(size_t)c * 7 * kD + i];
  if (which == 0) { db_ih[c_] += v_; db_hh[c_] += v_; }
  else if (which == 1) { db_ih[kD + c_] += v_; db_hh[kD + c_] += v_; }
  else if (which == 2) db_ih[2 * kD + c_] += v_;
  else if (which == 3) db_hh[2 * kD + c_] += v_;
  else db_fold[(which - 4) * kD + c_] += v_;
}

}  // namespace tc2b

// workspace = [dgrad per-slice transposed weight images (384 KB)][q images x4][h image][wgrad partial sums: 2 x 74 x 384 x 128 fp32]
constexpr int kWgCtas = kNumSMs / 6;       // x 6 gate blocks = one CTA per SM
static size_t wg_partial_bytes() { return (size_t)2 * kWgCtas * tc2b::kWgPartialFloats * sizeof(float); }
int gru_tc2b_trace_enable(int on) {
  DDFA_CUDA(cudaMemcpyToSymbol(tcc::g_trace_on, &on, sizeof(int)));
  return DDFA_OK;
}
int gru_tc2b_trace_read(void *host, size_t bytes) {
  if (bytes > tcc::kTraceWords * sizeof(long long)) bytes = tcc::kTraceWords * sizeof(long long);
  DDFA_CUDA(cudaMemcpyFromSymbol(host, tcc::g_trace, bytes));
  return DDFA_OK;
}
// workspace: [dgrad3 packed weights 384 KB][h image][dh' * z plane (image-sized)][s image (fp32-s entry only)]
//            [wgrad partial sums][bias-gradient slots (deterministic mode; reserved in both modes)][q images x 4] x slots   (one slot, or one per time step when the weight-gradient GEMM of a
//            whole backward pass is batched into one launch)
static constexpr size_t kPackedTotal = tc2b::kD3PackedBytes;
static constexpr size_t kBiasSlotBytes = (size_t)tc2b::kBiasSlots * 7 * tcc::kD * sizeof(float);
static size_t bwd_fixed_bytes(int32_t N) { return kPackedTotal + 3 * tcc::image_bytes(N) + wg_partial_bytes() + kBiasSlotBytes; }
void *gru_tc2_bwd_s_image_scratch(void *workspace, int32_t N) { return static_cast<uint8_t *>(workspace) + kPackedTotal + 2 * tcc::image_bytes(N); }
size_t gru_tc2_bwd_workspace_bytes(int32_t N, int32_t slots) {
  return bwd_fixed_bytes(N) + (size_t)(slots < 1 ? 1 : slots) * 4 * tcc::image_bytes(N);
}


int gru_tc2_prepare_bwd(const float *w_fold, const float *w_hh, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (workspace == nullptr || workspace_bytes < kPackedTotal) {
    set_error("tcgen05 engine (bwd): workspace too small");
    return DDFA_ERR_WORKSPACE;
  }
  const int total = 4 * 3 * 64 * 16;
  tc2b::dgrad3_pack_kernel<<<(total + 127) / 128, 128, 0, stream>>>(w_fold, w_hh, static_cast<uint8_t *>(workspace));
  DDFA_CHECK_LAUNCH("tc2b::dgrad3_pack_kernel");
  chain_break();
  return DDFA_OK;
}

// dW' += sum of the per-CTA partial sums, dWhh likewise (closes a deferred weight-gradient accumulation)
int gru_tc2_bwd_finish(int32_t N, float *dw_fold, float *dw_hh, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (workspace == nullptr || workspace_bytes < gru_tc2_bwd_workspace_bytes(N, 1)) {
    set_error("tcgen05 engine (bwd finish): workspace too small");
    return DDFA_ERR_WORKSPACE;
  }
  float *partial = reinterpret_cast<float *>(static_cast<uint8_t *>(workspace) + kPackedTotal + 3 * tcc::image_bytes(N));
  const int n4 = (int)(tc2b::kWgPartialFloats / 4);
  tc2b::wgrad_reduce_kernel<<<dim3((n4 + 255) / 256, 2), 256, 0, stream>>>(partial, kWgCtas, dw_fold, dw_hh);
  DDFA_CHECK_LAUNCH("tc2b::wgrad_reduce_kernel");
  return DDFA_OK;
}

// Clusters of bwd_step_fused_kernel that fit on the device at once (one CTA per SM; queried once per instantiation)
template <bool HF32, bool CSRP>
static int bwd_fused_max_clusters(int *out) {
  static std::atomic<int> cached{0};
  int v = cached.load(std::memory_order_relaxed);
  if (v == 0) {
    DDFA_CUDA(cudaFuncSetAttribute(tc2b::bwd_step_fused_kernel<HF32, CSRP>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2b::kD3SmemAlloc));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kNumSMs / 4 * 4);
    cfg.blockDim = dim3(tc2b::kD3Threads);
    cfg.dynamicSmemBytes = tc2b::kD3SmemAlloc;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 4;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    DDFA_CUDA(cudaOccupancyMaxActiveClusters(&v, tc2b::bwd_step_fused_kernel<HF32, CSRP>, &cfg));
    if (v < 1) {
      set_error("tcgen05 engine (bwd): bwd_step_fused_kernel fits no 4-CTA cluster on this device");
      return DDFA_ERR_CUDA;
    }
    cached.store(v, std::memory_order_relaxed);
  }
  *out = v;
  return DDFA_OK;
}
int gru_tc2b_fused_max_clusters(int *out) { return bwd_fused_max_clusters<false, true>(out); }

// One cluster of 4 CTAs per 128-node tile, persistent: min(tiles, the clusters that fit) clusters.  Chained (PDL) under bit 4 of
// DDFA_TUNE_PDL_MASK, the bit of the gate backward whose place it takes at the head of the step.
template <bool HF32, bool CSRP>
static int launch_bwd_fused(int tiles, cudaStream_t stream, const float *dh_out, const float *h, const void *h_img_in, const void *gates_packed,
                            const int32_t *indptr, const float *ds_in, const int32_t *indptr_t, const int32_t *indices_t, int32_t N,
                            uint8_t *q_img, size_t img, const uint8_t *packed, float *ds, float *dh, float *db_fold, float *db_ih, float *db_hh,
                            float *bias_slots, int *ctas) {
  int clusters = 0;
  const int rc = bwd_fused_max_clusters<HF32, CSRP>(&clusters);
  if (rc != DDFA_OK) return rc;
  if (clusters > tiles) clusters = tiles;
  *ctas = clusters * 4;
  DDFA_REQUIRE(bias_slots == nullptr || *ctas <= tc2b::kBiasSlots, "tcgen05 engine (bwd): %d CTAs exceed the %d bias-gradient slots",
               *ctas, tc2b::kBiasSlots);
  // ds and dh leave the kernel as [64 x 32] boxes; encoded per call, so a captured graph keeps the addresses of its capture
  CUtensorMap tm_ds, tm_dh;
  int rc_map = tcc::encode_f32_rows_map(ds, N, tc2b::kOutBoxCols, tc2b::kOutBoxRows, CU_TENSOR_MAP_SWIZZLE_128B, &tm_ds);
  if (rc_map == DDFA_OK) rc_map = tcc::encode_f32_rows_map(dh, N, tc2b::kOutBoxCols, tc2b::kOutBoxRows, CU_TENSOR_MAP_SWIZZLE_128B, &tm_dh);
  if (rc_map != DDFA_OK) return rc_map;
  DDFA_CUDA(cudaFuncSetAttribute(tc2b::bwd_step_fused_kernel<HF32, CSRP>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2b::kD3SmemAlloc));
  DDFA_CUDA(launch_chain_cluster(4, 4, tc2b::bwd_step_fused_kernel<HF32, CSRP>, dim3(clusters * 4), dim3(tc2b::kD3Threads), tc2b::kD3SmemAlloc,
                                 stream, dh_out, h, static_cast<const uint8_t *>(h_img_in), static_cast<const uint2 *>(gates_packed), indptr,
                                 ds_in, ds_in ? indptr_t : nullptr, indices_t, N, q_img, img, packed, tm_ds, tm_dh, dh, db_fold, db_ih, db_hh,
                                 bias_slots, l2_hints()));
  DDFA_CHECK_LAUNCH("tc2b::bwd_step_fused_kernel");
  return DDFA_OK;
}

// wgrad_mode: 0 = immediate (dW += this step's contribution before returning), 1 = first step of a deferred accumulation
// (partials overwritten), 2 = further deferred step (partials accumulated); deferred passes end with gru_tc2_bwd_finish.
// wgrad_mode >= 16: keep this step's q images in workspace slot (wgrad_mode - 16) and run no weight-gradient GEMM now —
// gru_tc2_bwd_wgrad_batched does it for all kept steps in one launch.
// h_img_in: the activation image of h (kept from the forward pass) or NULL (then it is rebuilt inside the workspace).
// ds_in / indptr_t / indices_t: NULL, or the incoming gradient is dh_out + A^T ds_in (A^T as a CSR over the transposed graph)
int gru_tc2_step_bwd(const float *dh_out, const float *ds_in, const int32_t *indptr_t, const int32_t *indices_t, const float *h,
                     const void *h_img_in, const void *s_img, const float *gates, const void *gates_packed, const int32_t *indptr, int32_t N, float *ds, float *dh, float *dw_fold, float *db_fold, float *db_ih,
                     float *dw_hh, float *db_hh, void *workspace, size_t workspace_bytes, int wgrad_mode, cudaStream_t stream) {
  if (h == nullptr && h_img_in == nullptr) {
    set_error("tcgen05 engine (bwd): neither the fp32 h nor its activation image given");
    return DDFA_ERR_INVALID_ARG;
  }
  const int q_slot = wgrad_mode >= 16 ? wgrad_mode - 16 : 0;
  if (workspace == nullptr || workspace_bytes < gru_tc2_bwd_workspace_bytes(N, q_slot + 1)) {
    set_error("tcgen05 engine (bwd): workspace too small (%zu < %zu)", workspace_bytes, gru_tc2_bwd_workspace_bytes(N, q_slot + 1));
    return DDFA_ERR_WORKSPACE;
  }
  uint8_t *packed = static_cast<uint8_t *>(workspace);
  const size_t img = tcc::image_bytes(N);
  uint8_t *h_img_ws = packed + kPackedTotal;
  float *partial = reinterpret_cast<float *>(h_img_ws + 3 * img);
  float *bias_slots = deterministic() ? reinterpret_cast<float *>(h_img_ws + 3 * img + wg_partial_bytes()) : nullptr;
  int ctas = 0;      // CTAs of the step's first kernel (one bias slot each)
  uint8_t *q_img = packed + bwd_fixed_bytes(N) + (size_t)q_slot * 4 * img;
  const uint8_t *h_img = h_img_in ? static_cast<const uint8_t *>(h_img_in) : h_img_ws;
  const int tiles = (N + tcc::kTileM - 1) / tcc::kTileM;
  if (gates_packed && gate_bwd_tma()) {
    // packed saved state: gate backward and dgrad in one cluster kernel (dh' * z handed over through the rows of dh)
    const bool csrp = gate_bwd_tma() >= 2;
    int rc = DDFA_OK;
    if (h) rc = csrp ? launch_bwd_fused<true, true>(tiles, stream, dh_out, h, h_img_in, gates_packed, indptr, ds_in, indptr_t, indices_t, N, q_img, img, packed, ds, dh, db_fold, db_ih, db_hh, bias_slots, &ctas)
                     : launch_bwd_fused<true, false>(tiles, stream, dh_out, h, h_img_in, gates_packed, indptr, ds_in, indptr_t, indices_t, N, q_img, img, packed, ds, dh, db_fold, db_ih, db_hh, bias_slots, &ctas);
    else   rc = csrp ? launch_bwd_fused<false, true>(tiles, stream, dh_out, h, h_img_in, gates_packed, indptr, ds_in, indptr_t, indices_t, N, q_img, img, packed, ds, dh, db_fold, db_ih, db_hh, bias_slots, &ctas)
                     : launch_bwd_fused<false, false>(tiles, stream, dh_out, h, h_img_in, gates_packed, indptr, ds_in, indptr_t, indices_t, N, q_img, img, packed, ds, dh, db_fold, db_ih, db_hh, bias_slots, &ctas);
    if (rc != DDFA_OK) return rc;
  } else {
    // register-path gate backward, then dgrad3 (the fp32 saved state, and DDFA_TUNE_GATE_BWD_TMA = 0)
    const int64_t rows = (int64_t)tiles * tcc::kTileM;
    const int64_t want = (rows + tc2b::kGbWarps - 1) / tc2b::kGbWarps;
    const unsigned gb_grid = (unsigned)(want < tc2b::kBiasSlots ? want : tc2b::kBiasSlots);
    ctas = (int)gb_grid;
    float *dhz = reinterpret_cast<float *>(h_img_ws + img);
    DDFA_CUDA(launch_chain(4, tc2b::gate_bwd_image_kernel, dim3(gb_grid), dim3(32 * tc2b::kGbWarps), 0, stream, dh_out, h,
                           static_cast<const uint8_t *>(h_img_in), gates, static_cast<const uint4 *>(gates_packed), indptr, ds_in,
                           ds_in ? indptr_t : nullptr, indices_t, N, q_img, img, h_img_in ? nullptr : h_img_ws, dhz, db_fold, db_ih, db_hh,
                           bias_slots, l2_hints()));
    DDFA_CHECK_LAUNCH("tc2b::gate_bwd_image_kernel");
    DDFA_CUDA(cudaFuncSetAttribute(tc2b::dgrad3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2b::kD3SmemAlloc));
    int groups = kNumSMs / 4;
    if (groups > tiles) groups = tiles;
    DDFA_CUDA(launch_chain(8, tc2b::dgrad3_kernel, dim3(groups * 4), dim3(tc2b::kD3Threads), tc2b::kD3SmemAlloc, stream, q_img, img, dhz,
                           static_cast<const uint8_t *>(packed), N, ds, dh, l2_hints()));
    DDFA_CHECK_LAUNCH("tc2b::dgrad3_kernel");
  }
  if (bias_slots) {
    tc2b::bias_slots_reduce_kernel<<<7, 128, 0, stream>>>(bias_slots, ctas, db_fold, db_ih, db_hh);
    DDFA_CHECK_LAUNCH("tc2b::bias_slots_reduce_kernel");
  }
  DDFA_CUDA(cudaFuncSetAttribute(tc2b::wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2b::kWgSmemAlloc));
  if (wgrad_mode >= 16) return DDFA_OK;       // q images kept; the batched weight-gradient launch follows the last step
  // every one of the 74 x 2 CTAs writes its partial slot (zeros if it owns no tile), so the reduction can sum all of them
  tc2b::WgBatch one = {};
  one.s_img[0] = static_cast<const uint8_t *>(s_img);
  one.h_img[0] = h_img;
  one.steps = 1;
  tc2b::wgrad_kernel<<<dim3(kWgCtas, 6), tc2b::kWgThreads, tc2b::kWgSmemAlloc, stream>>>(q_img, img, 0, one, N, partial, wgrad_mode == 2 ? 0 : 1, 0);
  DDFA_CHECK_LAUNCH("tc2b::wgrad_kernel");
  if (wgrad_mode == 0) return gru_tc2_bwd_finish(N, dw_fold, dw_hh, workspace, workspace_bytes, stream);
  return DDFA_OK;
}

// dW' += sum_t [q_r q_z q_n]_t^T s_t, dWhh += sum_t [q_r q_z q_nr]_t^T h_t over the `steps` slots kept by gru_tc2_step_bwd
// (wgrad_mode = 16 + slot): ONE weight-gradient launch with K = steps x nodes, then the reduction of the per-CTA partials.
int gru_tc2_bwd_wgrad_batched(const void *const *s_imgs, const void *const *h_imgs, int32_t steps, int32_t N, float *dw_fold,
                              float *dw_hh, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (steps < 1 || steps > tc2b::kWgMaxSteps) {
    set_error("tcgen05 engine (batched wgrad): 1 <= steps <= %d required (got %d)", tc2b::kWgMaxSteps, steps);
    return DDFA_ERR_INVALID_ARG;
  }
  if (workspace == nullptr || workspace_bytes < gru_tc2_bwd_workspace_bytes(N, steps)) {
    set_error("tcgen05 engine (batched wgrad): workspace too small (%zu < %zu)", workspace_bytes, gru_tc2_bwd_workspace_bytes(N, steps));
    return DDFA_ERR_WORKSPACE;
  }
  uint8_t *packed = static_cast<uint8_t *>(workspace);
  const size_t img = tcc::image_bytes(N);
  float *partial = reinterpret_cast<float *>(packed + kPackedTotal + 3 * img);
  const uint8_t *q_img = packed + bwd_fixed_bytes(N);
  tc2b::WgBatch b = {};
  for (int t = 0; t < steps; ++t) {
    if (!s_imgs[t] || !h_imgs[t]) {
      set_error("tcgen05 engine (batched wgrad): NULL image pointer for step %d", t);
      return DDFA_ERR_INVALID_ARG;
    }
    b.s_img[t] = static_cast<const uint8_t *>(s_imgs[t]);
    b.h_img[t] = static_cast<const uint8_t *>(h_imgs[t]);
  }
  b.steps = steps;
  DDFA_CUDA(cudaFuncSetAttribute(tc2b::wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2b::kWgSmemAlloc));
  tc2b::wgrad_kernel<<<dim3(kWgCtas, 6), tc2b::kWgThreads, tc2b::kWgSmemAlloc, stream>>>(q_img, img, 4 * img, b, N, partial, 1, l2_hints());
  DDFA_CHECK_LAUNCH("tc2b::wgrad_kernel");
  return gru_tc2_bwd_finish(N, dw_fold, dw_hh, workspace, workspace_bytes, stream);
}

}  // namespace ddfa
