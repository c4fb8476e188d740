// K3 — CSR edge gather-sum:  out[v,:] = (acc ? out[v,:] : 0) + sum_{e in [indptr[v], indptr[v+1])} h[indices[e], :]
//
// Replaces DGL's update_all(fn.copy_u('h','m'), fn.sum('m','a')) (SpMM) inside GatedGraphConv
// (reference call site DDFA/code_gnn/models/flow_gnn/ggnn.py:95).  Run on the CSR of the
// transposed graph it is that op's backward.
//
// Bound: HBM bandwidth (zero FLOPs).  Algorithmic bytes per launch:
//     E*D*4 (source rows) + N*D*4 (write) + E*4 (indices) + (N+1)*4 (indptr)
//
// Mapping: a group of G = min(32, D/4) lanes owns RW*PASSES consecutive destination rows; one lane
// holds one 16-byte column chunk, so a D=128 fp32 row (512 B) is exactly one warp-wide
// ld.global.nc.v4.  The kernel is latency-bound (ncu r01a: long-scoreboard stalls dominate: the
// chain indptr -> indices -> rows is three dependent DRAM/L2 round trips), so the index side is
// hoisted: ONE coalesced load fetches all RW*PASSES+1 row pointers of the group, then up to
// NIDX*G neighbour ids are prefetched into registers, and only then the row phase starts: the
// neighbour rows are fetched in batches of UNROLL independent 128-bit loads (memory-level
// parallelism) and folded into per-row accumulators by a warp-uniform segmented reduction (row
// boundaries broadcast with shuffles), RW rows per pass.  No atomics; neighbour lists are sorted,
// so the fp32 summation order — and the result — is deterministic.
#include <cuda_bf16.h>
#include <stdlib.h>

#include "common.cuh"

namespace ddfa {

// bf16 hi/lo split for the activation images, two values per conversion (cvt.rn.bf16x2.f32 = F2FP.PACK_AB: converts and packs;
// the scalar F2F form is a quarter-rate instruction per value plus a shift/OR per pair).  Same values as tc_common.cuh split_bf16.
__device__ __forceinline__ uint32_t bf16x2_word(float lo_half, float hi_half) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo_half, hi_half);      // .x -> bits 0-15, .y -> bits 16-31
  return *reinterpret_cast<const uint32_t *>(&v);
}
__device__ __forceinline__ void split4_bf16x2(const float4 &x, uint2 &ph, uint2 &pl) {
  ph.x = bf16x2_word(x.x, x.y);
  ph.y = bf16x2_word(x.z, x.w);
  pl.x = bf16x2_word(x.x - __uint_as_float(ph.x << 16), x.y - __uint_as_float(ph.x & 0xffff0000u));
  pl.y = bf16x2_word(x.z - __uint_as_float(ph.y << 16), x.w - __uint_as_float(ph.y & 0xffff0000u));
}


template <int G, int CH, int RW, int UNROLL, int PASSES, int NIDX, int THREADS>
__global__ void __launch_bounds__(THREADS) gather_sum_kernel(const int32_t *__restrict__ indptr,
                                                             const int32_t *__restrict__ indices,
                                                             const float *__restrict__ h, int32_t N, int32_t D,
                                                             float *__restrict__ out, int accumulate) {
  constexpr int GROUPS_PER_WARP = 32 / G;
  constexpr int ROWS = RW * PASSES;
  static_assert(ROWS + 1 <= G, "row pointers of a group must fit its lanes");
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;                 // lane inside the group
  const int gbase = lane - gl;             // first lane of the group inside the warp
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << gbase);
  const int64_t warp_global = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t group = warp_global * GROUPS_PER_WARP + (lane / G);
  const int64_t v0 = group * ROWS;
  if (v0 >= N) return;
  const int nrows = (int)min((int64_t)ROWS, (int64_t)N - v0);

  // row pointers of the whole group: lane i holds indptr[v0+i], i <= nrows
  int32_t myptr = 0;
  if (gl <= nrows) myptr = __ldg(indptr + v0 + gl);
  const int32_t beg0 = __shfl_sync(gmask, myptr, gbase);
  const int32_t total = __shfl_sync(gmask, myptr, gbase + nrows) - beg0;
  // prefetch the first NIDX*G neighbour ids of the group (coalesced)
  int32_t pre[NIDX];
#pragma unroll
  for (int b = 0; b < NIDX; ++b) pre[b] = (b * G + gl < total) ? __ldg(indices + beg0 + b * G + gl) : 0;

#pragma unroll 1
  for (int p = 0; p < PASSES; ++p) {
    const int r0 = p * RW;
    if (r0 >= nrows) break;
    int32_t rend[RW];  // row end offsets (relative to beg0) of this pass's rows
#pragma unroll
    for (int r = 0; r < RW; ++r) rend[r] = __shfl_sync(gmask, myptr, gbase + min(r0 + r + 1, nrows)) - beg0;
    const int32_t pbeg = __shfl_sync(gmask, myptr, gbase + r0) - beg0;
    const int32_t pend = rend[RW - 1];

    float4 acc[RW][CH];
#pragma unroll
    for (int r = 0; r < RW; ++r)
#pragma unroll
      for (int c = 0; c < CH; ++c) acc[r][c] = make_float4(0.f, 0.f, 0.f, 0.f);

    for (int32_t b = pbeg; b < pend; b += UNROLL) {
      float4 v[UNROLL][CH];
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) {
        const int32_t pos = min(b + j, pend - 1);  // clamp: every lane runs the shuffles
        const int blk = pos / G, l = pos - blk * G;
        int32_t u = 0;
        bool found = false;
#pragma unroll
        for (int q = 0; q < NIDX; ++q) {
          const int32_t t = __shfl_sync(gmask, pre[q], gbase + l);
          if (blk == q) { u = t; found = true; }
        }
        if (!found) u = __ldg(indices + beg0 + pos);  // very long neighbour lists: direct (uniform) load
        if (b + j < pend) {
          const float *row = h + (int64_t)u * D;
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int col = (gl + c * G) * 4;
            v[j][c] = (col < D) ? ldg_nc_f4(row + col) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        } else {
#pragma unroll
          for (int c = 0; c < CH; ++c) v[j][c] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) {
        const int32_t pos = b + j;
        // uniform (per group) segmented accumulate: edge `pos` belongs to the first row with rend > pos
#pragma unroll
        for (int r = 0; r < RW; ++r) {
          const bool mine = (pos < rend[r]) && (r == 0 ? true : pos >= rend[r - 1]);
          if (mine) {
#pragma unroll
            for (int c = 0; c < CH; ++c) f4_add(acc[r][c], v[j][c]);
          }
        }
      }
    }

#pragma unroll
    for (int r = 0; r < RW; ++r) {
      if (r0 + r < nrows) {
        float *orow = out + (v0 + r0 + r) * D;
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const int col = (gl + c * G) * 4;
          if (col < D) {
            float4 a = acc[r][c];
            if (accumulate) f4_add(a, *reinterpret_cast<const float4 *>(orow + col));
            *reinterpret_cast<float4 *>(orow + col) = a;
          }
        }
      }
    }
  }
}

template <int G, int CH, int RW, int UNROLL, int PASSES, int NIDX, int THREADS>
static int launch_gather(const int32_t *indptr, const int32_t *indices, const float *h, int32_t N, int32_t D,
                         float *out, int accumulate, cudaStream_t stream) {
  constexpr int GROUPS_PER_WARP = 32 / G;
  constexpr int ROWS = RW * PASSES;
  const int64_t groups = ((int64_t)N + ROWS - 1) / ROWS;
  const int64_t warps = (groups + GROUPS_PER_WARP - 1) / GROUPS_PER_WARP;
  const int64_t blocks = (warps * 32 + THREADS - 1) / THREADS;
  gather_sum_kernel<G, CH, RW, UNROLL, PASSES, NIDX, THREADS><<<(unsigned)blocks, THREADS, 0, stream>>>(indptr, indices, h, N, D, out, accumulate);
  DDFA_CHECK_LAUNCH("gather_sum_kernel");
  return DDFA_OK;
}

// ---- D = 128, output as an activation image (tc_common.cuh) for the tcgen05 engine --------------------
// Same mapping as variant 9 (2 rows per pass, 2 passes, 4 row loads in flight, 128-thread CTAs); the sum of a
// row is split into bf16 hi/lo and stored as 8-byte pieces of the swizzled image (16 lanes fill one 128-byte
// image row).  Rows N .. ceil128(N)-1 are written as zeros (the weight-gradient GEMM sums over all 128 rows).
__global__ void __launch_bounds__(128) gather_sum_image_kernel(const int32_t *__restrict__ indptr,
                                                               const int32_t *__restrict__ indices,
                                                               const float *__restrict__ h, int32_t N,
                                                               uint8_t *__restrict__ out_img, float *__restrict__ out_f32) {
  constexpr int RW = 2, PASSES = 2, ROWS = RW * PASSES, UNROLL = 4, D = 128;
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t v0 = warp_global * ROWS;
  const int64_t Npad = ((int64_t)N + 127) / 128 * 128;
  pdl_launch_dependents();
  pdl_wait();     // before ANY global read: the CSR arrays may have been rebuilt in place for this step (common.cuh, PDL rules)
  if (v0 >= Npad) return;
  const int nrows = (int)min((int64_t)ROWS, Npad - v0);
  int32_t myptr = 0;
  if (lane <= nrows) myptr = __ldcg(indptr + min(v0 + lane, (int64_t)N));   // padded rows: empty neighbour list
  const int32_t beg0 = __shfl_sync(0xffffffffu, myptr, 0);
  const int32_t total = __shfl_sync(0xffffffffu, myptr, nrows) - beg0;
  const int32_t pre = (lane < total) ? __ldcg(indices + beg0 + lane) : 0;
#pragma unroll 1
  for (int p = 0; p < PASSES; ++p) {
    const int r0 = p * RW;
    if (r0 >= nrows) break;
    int32_t rend[RW];
#pragma unroll
    for (int r = 0; r < RW; ++r) rend[r] = __shfl_sync(0xffffffffu, myptr, min(r0 + r + 1, nrows)) - beg0;
    const int32_t pbeg = __shfl_sync(0xffffffffu, myptr, r0) - beg0;
    const int32_t pend = rend[RW - 1];
    float4 acc[RW];
#pragma unroll
    for (int r = 0; r < RW; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int32_t b = pbeg; b < pend; b += UNROLL) {
      float4 v[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) {
        const int32_t pos = min(b + j, pend - 1);
        int32_t u = __shfl_sync(0xffffffffu, pre, pos & 31);
        if (pos >= 32) u = __ldcg(indices + beg0 + pos);
        v[j] = (b + j < pend) ? __ldcg(reinterpret_cast<const float4 *>(h + (int64_t)u * D + lane * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) {
        const int32_t pos = b + j;
#pragma unroll
        for (int r = 0; r < RW; ++r) {
          const bool mine = (pos < rend[r]) && (r == 0 ? true : pos >= rend[r - 1]);
          if (mine) f4_add(acc[r], v[j]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RW; ++r) {
      if (r0 + r < nrows) {
        const int64_t node = v0 + r0 + r;
        // bf16 hi/lo split of 4 consecutive columns -> two 8-byte stores into the swizzled image
        uint2 ph, pl;
        split4_bf16x2(acc[r], ph, pl);
        const int col = lane * 4, row = (int)(node & 127);
        const size_t tile_off = (size_t)(node >> 7) * 65536;
        const uint32_t sw = (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + (((((col & 63) >> 3) ^ (row & 7)) & 7) << 4) + (col & 7) * 2);
        *reinterpret_cast<uint2 *>(out_img + tile_off + (size_t)((0 * 2 + (col >> 6)) * 16384) + sw) = ph;
        *reinterpret_cast<uint2 *>(out_img + tile_off + (size_t)((1 * 2 + (col >> 6)) * 16384) + sw) = pl;
        if (out_f32 && node < N) *reinterpret_cast<float4 *>(out_f32 + node * D + col) = acc[r];
      }
    }
  }
}

// ---- D = 128, input AND output as activation images ------------------------------------------------------------------------
// The same gather for the steps whose h_t exists only as its image (tcgen05 engine, t >= 1: the forward GRU kernel no longer
// writes an fp32 copy of h').  A node's image row is four 128-byte pieces [hi | lo] x [cols 0-63 | 64-127]; lane l fetches one
// 16-byte unit (8 bf16) of each of two pieces (mapping: see the kernel).
// G: row groups per warp.  The CSR data of a group is a chain of dependent loads (indptr -> indices -> rows); with G > 1 a warp walks
// G consecutive groups and keeps the chain pipelined: while it fetches the rows of group i, the neighbour ids of group i + 1 and the
// row pointers of group i + 2 are already in flight, so per group only the row fetch is exposed instead of three latencies
// (the one-group form sat at 3.1 TB/s of DRAM traffic with ~50 % of the warps resident: latency, not bandwidth).
template <int G>
__global__ void __launch_bounds__(128) gather_sum_image_src_kernel(const int32_t *__restrict__ indptr,
                                                                   const int32_t *__restrict__ indices,
                                                                   const uint8_t *__restrict__ h_img, int32_t N,
                                                                   uint8_t *__restrict__ out_img) {
  // A warp owns 4 consecutive destination rows per group; each HALF-warp sums two of them.  Lane j of a half owns columns 8 j .. 8 j + 7:
  // per neighbour it fetches that unit's hi and lo 16-byte pieces (un-swizzling by row & 7), adds them (exact in fp32: h = hi + lo)
  // and accumulates — so every lane ends with final sums, which it splits and stores as the two pieces of the output image.
  constexpr int ROWS = 4, UNROLL = 2;
  const int lane = threadIdx.x & 31;
  const int hf = lane >> 4, j = lane & 15;
  const uint32_t piece_off = (uint32_t)((j >> 3) * 16384), unit16 = (uint32_t)((j & 7) << 4);
  const int64_t warp_global = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t Npad = ((int64_t)N + 127) / 128 * 128;
  pdl_launch_dependents();
  pdl_wait();
  // row pointers of group i (lanes 0..ROWS; rows past N: empty neighbour list -> zeros) and its first 32 neighbour ids
  auto load_ptr = [&](int i) -> int32_t {
    const int64_t v = (warp_global * G + i) * ROWS;
    return (i < G && v < Npad && lane <= ROWS) ? __ldcg(indptr + min(v + lane, (int64_t)N)) : 0;
  };
  auto load_ids = [&](int32_t ptr) -> int32_t {
    const int32_t b0 = __shfl_sync(0xffffffffu, ptr, 0), tot = __shfl_sync(0xffffffffu, ptr, ROWS) - b0;
    return (lane < tot) ? __ldcg(indices + b0 + lane) : 0;
  };
  int32_t ptr_cur = load_ptr(0), ptr_next = load_ptr(1);
  int32_t pre_cur = load_ids(ptr_cur);
#pragma unroll 1
  for (int gi = 0; gi < G; ++gi) {
    const int64_t v0 = (warp_global * G + gi) * ROWS;
    if (v0 >= Npad) return;        // warp-uniform; Npad is a multiple of 4: a group's four rows are all inside the padded range
    const int32_t myptr = ptr_cur, pre = pre_cur;
    if (G > 1) {                   // keep the chain of the next groups in flight
      pre_cur = load_ids(ptr_next);
      ptr_cur = ptr_next;
      ptr_next = load_ptr(gi + 2);
    }
    const int32_t beg0 = __shfl_sync(0xffffffffu, myptr, 0);
    // this half's two rows: edges [hbeg, hmid) belong to row 2 hf, [hmid, hend) to row 2 hf + 1 (offsets relative to beg0)
    const int32_t hbeg = __shfl_sync(0xffffffffu, myptr, 2 * hf) - beg0;
    const int32_t hmid = __shfl_sync(0xffffffffu, myptr, 2 * hf + 1) - beg0;
    const int32_t hend = __shfl_sync(0xffffffffu, myptr, 2 * hf + 2) - beg0;
    const int32_t len_other = __shfl_xor_sync(0xffffffffu, hend - hbeg, 16);
    const int32_t trips = max(hend - hbeg, len_other);       // warp-uniform trip count (the shuffles below need all lanes)
    float acc[2][8];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[r][i] = 0.f;
    for (int32_t t = 0; t < trips; t += UNROLL) {
      uint4 vh[UNROLL], vl[UNROLL];
#pragma unroll
      for (int q = 0; q < UNROLL; ++q) {
        const int32_t pos = hbeg + t + q;
        const bool on = pos < hend;
        const int32_t pc = on ? pos : 0;
        int32_t u = __shfl_sync(0xffffffffu, pre, pc & 31);
        if (on && pc >= 32) u = __ldcg(indices + beg0 + pc);
        const uint8_t *src = h_img + (size_t)(u >> 7) * 65536 + (size_t)(u & 127) * 128 + piece_off + (unit16 ^ (uint32_t)((u & 7) << 4));
        vh[q] = on ? __ldcg(reinterpret_cast<const uint4 *>(src)) : make_uint4(0u, 0u, 0u, 0u);
        vl[q] = on ? __ldcg(reinterpret_cast<const uint4 *>(src + 32768)) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int q = 0; q < UNROLL; ++q) {
        const int32_t pos = hbeg + t + q;
        const uint32_t wh[4] = {vh[q].x, vh[q].y, vh[q].z, vh[q].w}, wl[4] = {vl[q].x, vl[q].y, vl[q].z, vl[q].w};
        float x[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          x[2 * i] = __uint_as_float(wh[i] << 16) + __uint_as_float(wl[i] << 16);
          x[2 * i + 1] = __uint_as_float(wh[i] & 0xffff0000u) + __uint_as_float(wl[i] & 0xffff0000u);
        }
        if (pos < hmid) {
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[0][i] += x[i];
        } else if (pos < hend) {
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[1][i] += x[i];
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int64_t node = v0 + 2 * hf + r;
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        hw[i] = bf16x2_word(acc[r][2 * i], acc[r][2 * i + 1]);
        lw[i] = bf16x2_word(acc[r][2 * i] - __uint_as_float(hw[i] << 16), acc[r][2 * i + 1] - __uint_as_float(hw[i] & 0xffff0000u));
      }
      uint8_t *dst = out_img + (size_t)(node >> 7) * 65536 + (size_t)(node & 127) * 128 + piece_off + (unit16 ^ (uint32_t)((node & 7) << 4));
      *reinterpret_cast<uint4 *>(dst) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      *reinterpret_cast<uint4 *>(dst + 32768) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
  }
}

// Tuning variants for the D=128 case (selected by ddfa_gather_sum_variant / $DDFA_GATHER_VARIANT):
//   id : RW UNROLL PASSES NIDX THREADS
static int launch_d128_variant(int variant, const int32_t *indptr, const int32_t *indices, const float *h, int32_t N,
                               float *out, int accumulate, cudaStream_t stream) {
  switch (variant) {
    case 0: return launch_gather<32, 1, 4, 8, 1, 1, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 1: return launch_gather<32, 1, 4, 8, 2, 1, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 2: return launch_gather<32, 1, 4, 8, 4, 2, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 3: return launch_gather<32, 1, 4, 8, 4, 2, 128>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 4: return launch_gather<32, 1, 2, 4, 4, 1, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 5: return launch_gather<32, 1, 2, 4, 8, 2, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 6: return launch_gather<32, 1, 2, 8, 4, 1, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 7: return launch_gather<32, 1, 1, 4, 8, 1, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 8: return launch_gather<32, 1, 4, 4, 2, 1, 256>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 9: return launch_gather<32, 1, 2, 4, 2, 1, 128>(indptr, indices, h, N, 128, out, accumulate, stream);
    case 10:      // gather_tma.cu: neighbour rows staged in shared memory by per-row TMA bulk copies
    case 11:      // gather_tma.cu: ... by tensor-map tile copies (one row per copy)
      return launch_gather_tma(variant, indptr, indices, h, N, out, accumulate, stream);
    default:
      set_error("ddfa_gather_sum_variant: unknown variant %d (0..11)", variant);
      return DDFA_ERR_INVALID_ARG;
  }
}

static int default_variant() { return gather_variant(); }

static int check_gather_args(const int32_t *indptr, const int32_t *indices, const float *h, int32_t N, int32_t D, float *out) {
  DDFA_REQUIRE(N >= 0 && D > 0 && D % 4 == 0 && D <= 1024, "ddfa_gather_sum: unsupported shape N=%d D=%d (need D%%4==0, D<=1024)", N, D);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(indptr && indices && h && out, "ddfa_gather_sum: NULL pointer");
  DDFA_REQUIRE(aligned16(h) && aligned16(out), "ddfa_gather_sum: h/out must be 16-byte aligned");
  DDFA_REQUIRE(h != out, "ddfa_gather_sum: in-place gather is not supported");
  return DDFA_OK;
}

}  // namespace ddfa

extern "C" {

int ddfa_gather_sum(const int32_t *indptr, const int32_t *indices, const float *h, int32_t N, int32_t D, float *out,
                    int accumulate, void *stream_) {
  using namespace ddfa;
  int rc = check_gather_args(indptr, indices, h, N, D, out);
  if (rc || N == 0) return rc;
  cudaStream_t stream = as_stream(stream_);
  const int chunks = D / 4;  // 16-byte chunks per row
  if (D == 128) return launch_d128_variant(default_variant(), indptr, indices, h, N, out, accumulate, stream);
  if (chunks <= 8) return launch_gather<8, 1, 4, 8, 1, 1, 256>(indptr, indices, h, N, D, out, accumulate, stream);
  if (chunks <= 16) return launch_gather<16, 1, 4, 8, 2, 1, 256>(indptr, indices, h, N, D, out, accumulate, stream);
  if (chunks <= 32) return launch_gather<32, 1, 4, 8, 2, 1, 256>(indptr, indices, h, N, D, out, accumulate, stream);
  if (chunks <= 64) return launch_gather<32, 2, 2, 8, 2, 1, 256>(indptr, indices, h, N, D, out, accumulate, stream);
  if (chunks <= 128) return launch_gather<32, 4, 2, 4, 2, 1, 256>(indptr, indices, h, N, D, out, accumulate, stream);
  return launch_gather<32, 8, 1, 4, 2, 1, 256>(indptr, indices, h, N, D, out, accumulate, stream);
}

int ddfa_gather_sum_image(const int32_t *indptr, const int32_t *indices, const float *h, int32_t N, int32_t D,
                          void *out_image, float *out_f32, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gather_sum_image: activation images exist for D == 128 only (N=%d D=%d)", N, D);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(indptr && indices && h && out_image && aligned16(h) && aligned16(out_image), "ddfa_gather_sum_image: NULL or unaligned pointer");
  const int64_t rows = ((int64_t)N + 127) / 128 * 128;
  const int64_t warps = (rows + 3) / 4;
  const int64_t blocks = (warps * 32 + 127) / 128;
  DDFA_CUDA(launch_chain(1, gather_sum_image_kernel, dim3((unsigned)blocks), dim3(128), 0, as_stream(stream_), indptr, indices, h, N,
                         static_cast<uint8_t *>(out_image), out_f32));
  DDFA_CHECK_LAUNCH("gather_sum_image_kernel");
  return DDFA_OK;
}

int ddfa_gather_sum_image_src(const int32_t *indptr, const int32_t *indices, const void *h_image, int32_t N, int32_t D,
                              void *out_image, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gather_sum_image_src: activation images exist for D == 128 only (N=%d D=%d)", N, D);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(indptr && indices && h_image && out_image && aligned16(h_image) && aligned16(out_image) && h_image != out_image,
               "ddfa_gather_sum_image_src: NULL, unaligned or aliased pointer");
  const int64_t rows = ((int64_t)N + 127) / 128 * 128;
  // groups of 4 rows per warp (CSR chain pipelined across a warp's groups): measured neutral against one group per warp at C1 and
  // C0 (profiles/r04d_ab_gather_src_groups_*.log: the kernel is not bound by that chain), so the default stays one group
  const int g = gather_src_groups() > 0 ? gather_src_groups() : 1;
  const int64_t warps = (rows / 4 + g - 1) / g;
  const int64_t blocks = (warps * 32 + 127) / 128;
#define DDFA_GSRC(GG)                                                                                                                   \
  DDFA_CUDA(launch_chain(1, gather_sum_image_src_kernel<GG>, dim3((unsigned)blocks), dim3(128), 0, as_stream(stream_), indptr, indices, \
                         static_cast<const uint8_t *>(h_image), N, static_cast<uint8_t *>(out_image)))
  if (g >= 4) DDFA_GSRC(4);
  else if (g == 2) DDFA_GSRC(2);
  else DDFA_GSRC(1);
#undef DDFA_GSRC
  DDFA_CHECK_LAUNCH("gather_sum_image_src_kernel");
  return DDFA_OK;
}

int ddfa_gather_sum_variant(int variant, const int32_t *indptr, const int32_t *indices, const float *h, int32_t N,
                            int32_t D, float *out, int accumulate, void *stream_) {
  using namespace ddfa;
  int rc = check_gather_args(indptr, indices, h, N, D, out);
  if (rc || N == 0) return rc;
  DDFA_REQUIRE(D == 128, "ddfa_gather_sum_variant: tuning variants exist for D == 128 only (got %d)", D);
  return launch_d128_variant(variant, indptr, indices, h, N, out, accumulate, as_stream(stream_));
}

}  // extern "C"
