// label_style="node" training: the rows the loss is taken over, drawn on the device, and the MLP head + BCE over that row list.
//
// Reference: BaseModule.resample (base_module.py:96-137: every vulnerable node plus round(#vulnerable * factor) non-vulnerable
// ones from random.sample) and the node-style loss (base_module.py:84-85,178-183: BCEWithLogitsLoss(pos_weight), mean over the
// kept rows).  The module path (module.py) keeps the host-side draw; these entry points serve FusedTrainer, whose step is one
// captured CUDA graph: nothing here syncs with the host, and every grid is sized from the node capacity N with the row count S
// read on the device.
//
// Sampling: the non-vulnerable valid nodes get a Philox4x32-10 key each, and the draw is the k smallest (key, node) pairs —
// a uniform k-subset.  The k-th smallest key is found by a radix select, 8 bits per pass (four multi-CTA histogram passes with
// integer atomics, each followed by a one-CTA bin pick); ties at that key are taken in node order.  The row list is then
// compacted in ascending node order by a block-count / scan / write sequence.  Integer counts only: the result does not depend on
// the order in which CTAs run.
//
// Several ranks (ddfa_node_dp_*): the same kernels, run in phases over one rank's shard of a global batch, with the caller's SUM
// exchanges between them: per-rank counts, the digit histograms (written to the exchange buffer instead of the workspace) and the
// tie counts.  Keys are those of node kOff + n of the global batch (kOff = 0 on one rank) and the block scan takes the ties of
// the ranks before this one first, so the union of the ranks' rows is ddfa_node_sample's row list of the concatenated batch.
//
// Head: SIMT fp32 (FFMA), so every hidden width works.  Hidden layers are 64 x 64-tiled GEMMs over the row list (layer 0 gathers
// [h_T[r] | x[r]] straight from the two planes); the last layer is a warp per row.  Weight and bias gradients are reduced over the
// rows in a fixed order in both tuning modes: kHeadChunks private partials over fixed row chunks, added in chunk order.
#include <math.h>

#include "common.cuh"

namespace ddfa {
namespace node {

constexpr int kThreads = 256;
constexpr int kPerThread = 4;                        // consecutive nodes per thread in the sampler
constexpr int kPerBlock = kThreads * kPerThread;     // nodes per sampler CTA
constexpr int kCtl = 16;                             // control words at the head of the sampler workspace
constexpr int kBins = 256;
constexpr int kHeadChunks = 32;                      // row chunks of the weight-gradient reduction
constexpr int kMaxLayers = 16;

// control words
// kOff: the node offset of this rank's shard in the global batch (0 on one rank): node n's key is that of node kOff + n
enum { kNVuln = 0, kPop = 1, kK = 2, kPrefix = 3, kKRem = 4, kDrawLo = 5, kDrawHi = 6, kOff = 7 };

inline int32_t num_blocks(int32_t N) { return (N + kPerBlock - 1) / kPerBlock; }

// Philox4x32-10 (Salmon et al., SC'11): counter (draw, node), key = the 64-bit seed; the first output word is the node's key
__device__ __forceinline__ uint32_t philox_key(uint32_t draw_lo, uint32_t draw_hi, uint32_t node, uint64_t seed) {
  uint32_t c0 = draw_lo, c1 = draw_hi, c2 = node, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return c0;
}

__device__ __forceinline__ int32_t valid_count(const int32_t *num_valid, int32_t N) { return min(max(*num_valid, 0), N); }

// exclusive block-wide prefix sum of one int per thread (kThreads threads); *total = the sum
__device__ __forceinline__ int32_t block_scan(int32_t v, int32_t *total) {
  __shared__ int32_t s_warp[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int32_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int32_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const int32_t t = s_warp[w];
    before += (w < warp) ? t : 0;
    all += t;
  }
  __syncthreads();     // s_warp is reused by the next call
  *total = all;
  return before + inc - v;
}

// no undersampling: every valid node, in order
__global__ void __launch_bounds__(kThreads) sample_all_kernel(const int32_t *__restrict__ num_valid, int32_t N, int32_t *__restrict__ rows,
                                                              int32_t *__restrict__ num_rows) {
  const int32_t nv = valid_count(num_valid, N);
  const int64_t n = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  if (n < nv) rows[n] = (int32_t)n;
  if (n == 0) *num_rows = nv;
}

// #vulnerable and #non-vulnerable valid nodes
__global__ void __launch_bounds__(kThreads) sample_count_kernel(const int32_t *__restrict__ vuln, const int32_t *__restrict__ num_valid, int32_t N,
                                                                int32_t *__restrict__ ctl) {
  const int32_t nv = valid_count(num_valid, N);
  int32_t nvul = 0, npop = 0;
  for (int64_t n = blockIdx.x * (int64_t)kThreads + threadIdx.x; n < nv; n += (int64_t)gridDim.x * kThreads) {
    if (vuln[n] != 0) ++nvul;
    else ++npop;
  }
  int32_t tv, tp;
  block_scan(nvul, &tv);
  block_scan(npop, &tp);
  if (threadIdx.x == 0) {
    if (tv) atomicAdd(ctl + kNVuln, tv);
    if (tp) atomicAdd(ctl + kPop, tp);
  }
}

// k = rint(n_vuln * factor) in fp64 (Python's round() of the same product), clamped to the population with the status word set;
// takes this call's draw index and advances the caller's counter
__device__ __forceinline__ void draw_size(int32_t *__restrict__ ctl, double factor, int64_t *__restrict__ draw, int32_t *__restrict__ status) {
  const double want = rint((double)ctl[kNVuln] * factor);
  const int32_t pop = ctl[kPop];
  int32_t k;
  if (!(want <= (double)pop)) {      // also NaN / inf
    k = pop;
    *status = 1;
  } else {
    k = (int32_t)want;
  }
  ctl[kK] = k;
  ctl[kKRem] = k;
  ctl[kPrefix] = 0;
  const int64_t d = *draw;
  ctl[kDrawLo] = (int32_t)(uint32_t)(uint64_t)d;
  ctl[kDrawHi] = (int32_t)(uint32_t)((uint64_t)d >> 32);
  *draw = d + 1;
}

__global__ void sample_k_kernel(int32_t *__restrict__ ctl, double factor, int64_t *__restrict__ draw, int32_t *__restrict__ status) {
  draw_size(ctl, factor, draw, status);
}

// several ranks: counts[2q..2q+2) = [n_vuln, n_pop] of rank q (summed over the ranks by the caller's exchange).  The global counts
// and this rank's node offset go into ctl, then k / status / draw as on one rank; num_rows_global = S of the global batch
__global__ void dp_plan_kernel(const int32_t *__restrict__ counts, int32_t rank, int32_t world, double factor, int64_t *__restrict__ draw,
                               int32_t *__restrict__ status, int32_t *__restrict__ ctl, int32_t *__restrict__ num_rows_global,
                               int32_t *__restrict__ node_offset) {
  int32_t nvul = 0, pop = 0, off = 0;
  for (int32_t q = 0; q < world; ++q) {
    nvul += counts[2 * q];
    pop += counts[2 * q + 1];
    if (q < rank) off += counts[2 * q] + counts[2 * q + 1];
  }
  *node_offset = off;
  if (!(factor >= 0.0)) {      // no undersampling: every valid node of every rank
    *num_rows_global = nvul + pop;
    return;
  }
  ctl[kNVuln] = nvul;
  ctl[kPop] = pop;
  ctl[kOff] = off;
  draw_size(ctl, factor, draw, status);
  *num_rows_global = nvul + ctl[kK];
}

// histogram of digit `pass` over the candidates whose higher digits equal the prefix picked so far
__global__ void __launch_bounds__(kThreads) radix_hist_kernel(const int32_t *__restrict__ vuln, const int32_t *__restrict__ num_valid, int32_t N,
                                                              uint64_t seed, int pass, int32_t *__restrict__ ctl, uint32_t *__restrict__ hist) {
  __shared__ uint32_t s_hist[kBins];
  if (ctl[kK] == 0) return;
  s_hist[threadIdx.x] = 0u;
  __syncthreads();
  const int32_t nv = valid_count(num_valid, N);
  const uint32_t dlo = (uint32_t)ctl[kDrawLo], dhi = (uint32_t)ctl[kDrawHi], prefix = (uint32_t)ctl[kPrefix], off = (uint32_t)ctl[kOff];
  const int shift = 24 - 8 * pass;
  for (int64_t n = blockIdx.x * (int64_t)kThreads + threadIdx.x; n < nv; n += (int64_t)gridDim.x * kThreads) {
    if (vuln[n] != 0) continue;
    const uint32_t key = philox_key(dlo, dhi, off + (uint32_t)n, seed);
    if (pass > 0 && (key >> (shift + 8)) != (prefix >> (shift + 8))) continue;
    atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
  }
  __syncthreads();
  const uint32_t c = s_hist[threadIdx.x];
  if (c) atomicAdd(hist + threadIdx.x, c);
}

// the bin that holds the k_rem-th smallest candidate: its digit goes into the prefix, k_rem becomes the rank inside it; clears
// the histogram for the next pass
__global__ void __launch_bounds__(kBins) radix_pick_kernel(int pass, int32_t *__restrict__ ctl, uint32_t *__restrict__ hist) {
  if (ctl[kK] == 0) return;
  __shared__ uint32_t s_hist[kBins];
  s_hist[threadIdx.x] = hist[threadIdx.x];
  __syncthreads();
  hist[threadIdx.x] = 0u;
  if (threadIdx.x == 0) {
    const uint32_t want = (uint32_t)ctl[kKRem];
    uint32_t cum = 0u;
    for (int b = 0; b < kBins; ++b) {
      if (cum + s_hist[b] >= want) {
        ctl[kPrefix] = (int32_t)((uint32_t)ctl[kPrefix] | ((uint32_t)b << (24 - 8 * pass)));
        ctl[kKRem] = (int32_t)(want - cum);
        break;
      }
      cum += s_hist[b];
    }
  }
}

// node n's class: 2 = in the list for sure (vulnerable, or key below the threshold), 1 = tie at the threshold key, 0 = out
__device__ __forceinline__ int node_class(const int32_t *__restrict__ vuln, int32_t n, int32_t nv, uint32_t dlo, uint32_t dhi, uint32_t off,
                                          uint64_t seed, uint32_t thresh, bool any) {
  if (n >= nv) return 0;
  if (vuln[n] != 0) return 2;
  if (!any) return 0;
  const uint32_t key = philox_key(dlo, dhi, off + (uint32_t)n, seed);
  return key < thresh ? 2 : (key == thresh ? 1 : 0);
}

// per CTA: #sure rows and #ties (blk[0..nb) / blk[nb..2nb))
__global__ void __launch_bounds__(kThreads) sample_block_count_kernel(const int32_t *__restrict__ vuln, const int32_t *__restrict__ num_valid,
                                                                      int32_t N, uint64_t seed, const int32_t *__restrict__ ctl,
                                                                      int32_t *__restrict__ blk) {
  const int32_t nv = valid_count(num_valid, N);
  const uint32_t dlo = (uint32_t)ctl[kDrawLo], dhi = (uint32_t)ctl[kDrawHi], thresh = (uint32_t)ctl[kPrefix], off = (uint32_t)ctl[kOff];
  const bool any = ctl[kK] > 0;
  int32_t sure = 0, tie = 0;
  const int32_t n0 = blockIdx.x * kPerBlock + threadIdx.x * kPerThread;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    const int c = node_class(vuln, n0 + j, nv, dlo, dhi, off, seed, thresh, any);
    sure += c == 2;
    tie += c == 1;
  }
  int32_t ts, tt;
  block_scan(sure, &ts);
  block_scan(tie, &tt);
  if (threadIdx.x == 0) {
    blk[blockIdx.x] = ts;
    blk[gridDim.x + blockIdx.x] = tt;
  }
}

// one CTA, in CTA order: blk[2nb..3nb) = ties before each CTA, blk[3nb..4nb) = rows before each CTA; S.  Several ranks:
// rank_ties[q] = the ties of rank q, and the ties of ranks q < rank come before this rank's (NULL: one rank)
__global__ void __launch_bounds__(kThreads) sample_block_scan_kernel(int32_t nb, const int32_t *__restrict__ ctl, int32_t *__restrict__ blk,
                                                                     int32_t *__restrict__ num_rows, const int32_t *__restrict__ rank_ties,
                                                                     int32_t rank) {
  const int32_t take = ctl[kK] > 0 ? ctl[kKRem] : 0;
  int32_t tie_carry = 0, row_carry = 0;
  if (rank_ties)
    for (int32_t q = 0; q < rank; ++q) tie_carry += rank_ties[q];
  for (int32_t b0 = 0; b0 < nb; b0 += kThreads) {
    const int32_t b = b0 + threadIdx.x;
    const int32_t sure = b < nb ? blk[b] : 0, tie = b < nb ? blk[nb + b] : 0;
    int32_t tt;
    const int32_t tie_off = tie_carry + block_scan(tie, &tt);
    const int32_t mine = sure + min(max(take - tie_off, 0), tie);
    int32_t tr;
    const int32_t row_off = row_carry + block_scan(mine, &tr);
    if (b < nb) {
      blk[2 * nb + b] = tie_off;
      blk[3 * nb + b] = row_off;
    }
    tie_carry += tt;
    row_carry += tr;
  }
  if (threadIdx.x == 0) *num_rows = row_carry;
}

// this rank's ties at the threshold key: the sum of blk[nb..2nb)
__global__ void __launch_bounds__(kThreads) tie_total_kernel(int32_t nb, const int32_t *__restrict__ blk, int32_t *__restrict__ out) {
  int32_t acc = 0;
  for (int32_t b = threadIdx.x; b < nb; b += kThreads) acc += blk[nb + b];
  int32_t total;
  block_scan(acc, &total);
  if (threadIdx.x == 0) *out = total;
}

__global__ void __launch_bounds__(kThreads) sample_write_kernel(const int32_t *__restrict__ vuln, const int32_t *__restrict__ num_valid, int32_t N,
                                                                uint64_t seed, const int32_t *__restrict__ ctl, const int32_t *__restrict__ blk,
                                                                int32_t *__restrict__ rows) {
  const int32_t nb = gridDim.x;
  const int32_t nv = valid_count(num_valid, N);
  const uint32_t dlo = (uint32_t)ctl[kDrawLo], dhi = (uint32_t)ctl[kDrawHi], thresh = (uint32_t)ctl[kPrefix], off = (uint32_t)ctl[kOff];
  const bool any = ctl[kK] > 0;
  const int32_t take = any ? ctl[kKRem] : 0;
  const int32_t n0 = blockIdx.x * kPerBlock + threadIdx.x * kPerThread;
  int cls[kPerThread];
  int32_t tie = 0;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    cls[j] = node_class(vuln, n0 + j, nv, dlo, dhi, off, seed, thresh, any);
    tie += cls[j] == 1;
  }
  int32_t total;
  int32_t tie_rank = blk[2 * nb + blockIdx.x] + block_scan(tie, &total);
  int32_t mine = 0;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    if (cls[j] == 1) cls[j] = (tie_rank++ < take) ? 2 : 0;
    mine += cls[j] == 2;
  }
  int32_t pos = blk[3 * nb + blockIdx.x] + block_scan(mine, &total);
#pragma unroll
  for (int j = 0; j < kPerThread; ++j)
    if (cls[j] == 2) rows[pos++] = n0 + j;
}

// ---- head --------------------------------------------------------------------------------------------------------------
constexpr int BM = 64, BN = 64, BK = 16;
enum Epi { kBiasRelu = 0, kMask = 1, kScatter = 2 };

// A[s, k] of the row list: [h_T[rows[s]] | x[rows[s]]] (Gather) or a compact [S, K] matrix
template <bool Gather>
__device__ __forceinline__ float load_a(const float *__restrict__ a, const float *__restrict__ h, const float *__restrict__ x,
                                        const int32_t *__restrict__ rows, int32_t D, int32_t K, int32_t s, int32_t k) {
  if constexpr (Gather) {
    const int64_t r = rows[s];
    return k < D ? h[r * D + k] : x[r * D + (k - D)];
  } else {
    return a[(int64_t)s * K + k];
  }
}

// C[s, j] = sum_k A[s, k] * B(k, j) over the rows s < S, B(k, j) = TransB ? b[j * K + k] : b[k * Nout + j]; then the epilogue:
// kBiasRelu out = relu(C + bias) (compact [S, Nout]); kMask out = mask <= 0 ? 0 : C (compact); kScatter C into the two planes
// dh (columns < D) and dx (columns >= D) at row rows[s]
template <bool Gather, bool TransB, int E>
__global__ void __launch_bounds__(256) head_gemm_kernel(const float *__restrict__ a, const float *__restrict__ h, const float *__restrict__ x,
                                                        const int32_t *__restrict__ rows, const int32_t *__restrict__ num_rows, int32_t D,
                                                        int32_t K, int32_t Nout, const float *__restrict__ b, const float *__restrict__ bias,
                                                        const float *__restrict__ mask, float *__restrict__ out, float *__restrict__ dh,
                                                        float *__restrict__ dx) {
  const int32_t S = *num_rows;
  const int32_t s0 = blockIdx.x * BM, j0 = blockIdx.y * BN;
  if (s0 >= S) return;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4] = {};
  for (int32_t k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + 256 * i;
      const int m = e >> 4, kk = e & 15;
      const int32_t s = s0 + m, k = k0 + kk;
      As[kk][m] = (s < S && k < K) ? load_a<Gather>(a, h, x, rows, D, K, s, k) : 0.f;
      int jj, kb;
      if constexpr (TransB) { jj = e >> 4; kb = e & 15; }
      else { kb = e >> 6; jj = e & 63; }
      const int32_t j = j0 + jj, kg = k0 + kb;
      float bv = 0.f;
      if (j < Nout && kg < K) bv = TransB ? b[(int64_t)j * K + kg] : b[(int64_t)kg * Nout + j];
      Bs[kb][jj] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[kk][ty * 4 + i]; bv[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int32_t s = s0 + ty * 4 + i;
    if (s >= S) continue;
    const int64_t r = E == kScatter ? (int64_t)rows[s] : 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int32_t c = j0 + tx * 4 + j;
      if (c >= Nout) continue;
      const float v = acc[i][j];
      if constexpr (E == kBiasRelu) out[(int64_t)s * Nout + c] = relu_nan(v + bias[c]);
      else if constexpr (E == kMask) out[(int64_t)s * Nout + c] = relu_grad(mask[(int64_t)s * Nout + c], v);
      else {
        if (c < D) dh[r * D + c] = v;
        else dx[r * D + (c - D)] = v;
      }
    }
  }
}

// the last layer, Linear(K, 1): a warp per row
template <bool Gather>
__global__ void __launch_bounds__(256) head_out_kernel(const float *__restrict__ a, const float *__restrict__ h, const float *__restrict__ x,
                                                       const int32_t *__restrict__ rows, const int32_t *__restrict__ num_rows, int32_t D,
                                                       int32_t K, const float *__restrict__ w, const float *__restrict__ bias,
                                                       float *__restrict__ logits) {
  const int32_t S = *num_rows;
  const int lane = threadIdx.x & 31;
  const int32_t s = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  float acc = 0.f;
  for (int32_t k = lane; k < K; k += 32) acc = fmaf(load_a<Gather>(a, h, x, rows, D, K, s, k), w[k], acc);
  acc = warp_sum(acc);
  if (lane == 0) logits[s] = acc + bias[0];
}

// d input of the last layer: dlogits[s] * w[k], masked by the previous layer's ReLU (compact out) or scattered into the planes
template <bool Scatter>
__global__ void __launch_bounds__(256) head_last_bwd_kernel(const float *__restrict__ dlogits, const float *__restrict__ w,
                                                            const float *__restrict__ mask, const int32_t *__restrict__ rows,
                                                            const int32_t *__restrict__ num_rows, int32_t D, int32_t N, float *__restrict__ out,
                                                            float *__restrict__ dh, float *__restrict__ dx) {
  const int32_t S = *num_rows;
  const int32_t K = 2 * D;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)S * K) return;
  const int32_t s = (int32_t)(i / K), k = (int32_t)(i % K);
  const float v = dlogits[s] * w[k];
  if constexpr (Scatter) {
    const int64_t r = rows[s];
    if (k < D) dh[r * D + k] = v;
    else dx[r * D + (k - D)] = v;
  } else {
    out[i] = relu_grad(mask[i], v);
  }
}

// partial[c][j * K + k] = sum over the rows s of chunk c of dout[s, j] * in[s, k] (chunk = ceil(S / kHeadChunks) rows, in order);
// every CTA writes its tile, also when its chunk is empty
template <bool Gather>
__global__ void __launch_bounds__(256) head_wgrad_kernel(const float *__restrict__ dout, const float *__restrict__ a, const float *__restrict__ h,
                                                         const float *__restrict__ x, const int32_t *__restrict__ rows,
                                                         const int32_t *__restrict__ num_rows, int32_t D, int32_t K, int32_t Nout,
                                                         float *__restrict__ partial) {
  const int32_t S = *num_rows;
  const int32_t chunk = (S + kHeadChunks - 1) / kHeadChunks;
  const int c = blockIdx.z;
  const int32_t r0 = min(S, c * chunk), r1 = min(S, r0 + chunk);
  const int32_t j0 = blockIdx.y * BM, k0 = blockIdx.x * BN;
  __shared__ float Ds[BK][BM + 4];
  __shared__ float As[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4] = {};
  for (int32_t sb = r0; sb < r1; sb += BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + 256 * i;
      const int ss = e >> 6, cc = e & 63;
      const int32_t s = sb + ss;
      const bool in = s < r1;
      Ds[ss][cc] = (in && j0 + cc < Nout) ? dout[(int64_t)s * Nout + j0 + cc] : 0.f;
      As[ss][cc] = (in && k0 + cc < K) ? load_a<Gather>(a, h, x, rows, D, K, s, k0 + cc) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int ss = 0; ss < BK; ++ss) {
      float dv[4], av[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { dv[i] = Ds[ss][ty * 4 + i]; av[i] = As[ss][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(dv[i], av[j], acc[i][j]);
    }
    __syncthreads();
  }
  float *p = partial + (int64_t)c * Nout * K;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int32_t j = j0 + ty * 4 + i;
    if (j >= Nout) continue;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int32_t k = k0 + tx * 4 + jj;
      if (k < K) p[(int64_t)j * K + k] = acc[i][jj];
    }
  }
}

// bias partials: partial[c][j] = sum over chunk c's rows of dout[s, j], in row order
__global__ void __launch_bounds__(256) head_bias_partial_kernel(const float *__restrict__ dout, const int32_t *__restrict__ num_rows, int32_t Nout,
                                                                float *__restrict__ partial) {
  const int32_t S = *num_rows;
  const int32_t chunk = (S + kHeadChunks - 1) / kHeadChunks;
  const int c = blockIdx.y;
  const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= Nout) return;
  const int32_t r0 = min(S, c * chunk), r1 = min(S, r0 + chunk);
  float acc = 0.f;
  for (int32_t s = r0; s < r1; ++s) acc += dout[(int64_t)s * Nout + j];
  partial[(int64_t)c * Nout + j] = acc;
}

// out[i] += sum_c partial[c][i], c in order
__global__ void __launch_bounds__(256) chunk_reduce_kernel(const float *__restrict__ partial, int64_t n, float *__restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = 0.f;
#pragma unroll 8
  for (int c = 0; c < kHeadChunks; ++c) acc += partial[(int64_t)c * n + i];
  out[i] += acc;
}

// mean BCEWithLogits(pos_weight) over the S rows, one CTA in a fixed order (graph_label_bce_kernel's formula); S = 0 gives NaN.
// Scaled: the gradient's row scale is (1 / S) * grad_scale (gradient accumulation); the unscaled form never reads grad_scale.
// norm (several ranks): the sum over the S rows divided by *norm, the global row count, instead of S (NULL: by S)
template <bool Scaled>
__global__ void __launch_bounds__(1024) node_bce_kernel(const float *__restrict__ logits, const int32_t *__restrict__ vuln,
                                                        const int32_t *__restrict__ rows, const int32_t *__restrict__ num_rows,
                                                        const int32_t *__restrict__ norm, float pos_weight, float grad_scale,
                                                        float *__restrict__ loss_out, float *__restrict__ dlogits) {
  __shared__ float s_t[1024];
  const int32_t S = *num_rows;
  const float div = (float)(norm ? *norm : S);
  const float inv = Scaled ? (1.f / div) * grad_scale : 1.f / div;
  float acc = 0.f;
  for (int32_t s = threadIdx.x; s < S; s += 1024) {
    const float xv = logits[s], y = (float)vuln[rows[s]];
    const float lw = 1.f + (pos_weight - 1.f) * y;
    acc += (1.f - y) * xv + lw * (log1pf(expf(-fabsf(xv))) + fmaxf(-xv, 0.f));
    if (dlogits) dlogits[s] = inv * ((1.f - y) - lw * (1.f - 1.f / (1.f + expf(-xv))));
  }
  s_t[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_t[threadIdx.x] += s_t[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0 && loss_out) *loss_out = s_t[0] / div;
}

inline unsigned cdiv(int64_t a, int64_t b) { return (unsigned)((a + b - 1) / b); }

template <bool Gather>
int launch_wgrad(const float *dout, const float *a, const float *h, const float *x, const int32_t *rows, const int32_t *num_rows, int32_t D,
                 int32_t Nout, float *dw, float *db, float *partial, cudaStream_t stream) {
  const int32_t K = 2 * D;
  head_wgrad_kernel<Gather><<<dim3(cdiv(K, BN), cdiv(Nout, BM), kHeadChunks), 256, 0, stream>>>(dout, a, h, x, rows, num_rows, D, K, Nout, partial);
  DDFA_CHECK_LAUNCH("head_wgrad_kernel");
  chunk_reduce_kernel<<<cdiv((int64_t)Nout * K, 256), 256, 0, stream>>>(partial, (int64_t)Nout * K, dw);
  DDFA_CHECK_LAUNCH("chunk_reduce_kernel");
  head_bias_partial_kernel<<<dim3(cdiv(Nout, 256), kHeadChunks), 256, 0, stream>>>(dout, num_rows, Nout, partial);
  DDFA_CHECK_LAUNCH("head_bias_partial_kernel");
  chunk_reduce_kernel<<<cdiv(Nout, 256), 256, 0, stream>>>(partial, Nout, db);
  DDFA_CHECK_LAUNCH("chunk_reduce_kernel");
  return DDFA_OK;
}

}  // namespace node
}  // namespace ddfa

extern "C" {

size_t ddfa_node_sample_workspace_bytes(int32_t N) {
  using namespace ddfa::node;
  if (N < 0) return 0;
  return sizeof(int32_t) * ((size_t)kCtl + kBins + 4 * (size_t)num_blocks(N));
}

int ddfa_node_sample(const int32_t *vuln, const int32_t *num_valid, int32_t N, double factor, uint64_t seed, int64_t *draw, int32_t *rows,
                     int32_t *num_rows, int32_t *status, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  DDFA_REQUIRE(N >= 0, "ddfa_node_sample: num_nodes=%d < 0", N);
  DDFA_REQUIRE(num_valid && num_rows, "ddfa_node_sample: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  if (!(factor >= 0.0)) {       // no undersampling: every valid node
    DDFA_REQUIRE(N == 0 || rows, "ddfa_node_sample: NULL rows");
    sample_all_kernel<<<cdiv(N > 0 ? N : 1, kThreads), kThreads, 0, stream>>>(num_valid, N, rows, num_rows);
    DDFA_CHECK_LAUNCH("sample_all_kernel");
    return DDFA_OK;
  }
  DDFA_REQUIRE(vuln || N == 0, "ddfa_node_sample: NULL vuln");
  DDFA_REQUIRE(draw && status && workspace && (rows || N == 0), "ddfa_node_sample: NULL pointer");
  if (workspace_bytes < ddfa_node_sample_workspace_bytes(N)) {
    set_error("ddfa_node_sample: workspace too small (%zu < %zu)", workspace_bytes, ddfa_node_sample_workspace_bytes(N));
    return DDFA_ERR_WORKSPACE;
  }
  int32_t *ctl = static_cast<int32_t *>(workspace);
  uint32_t *hist = reinterpret_cast<uint32_t *>(ctl + kCtl);
  int32_t *blk = ctl + kCtl + kBins;
  const int32_t nb = num_blocks(N) > 0 ? num_blocks(N) : 1;
  const unsigned grid = (unsigned)min(nb, 4 * kNumSMs);
  DDFA_CUDA(cudaMemsetAsync(ctl, 0, sizeof(int32_t) * (kCtl + kBins), stream));
  sample_count_kernel<<<grid, kThreads, 0, stream>>>(vuln, num_valid, N, ctl);
  DDFA_CHECK_LAUNCH("sample_count_kernel");
  sample_k_kernel<<<1, 1, 0, stream>>>(ctl, factor, draw, status);
  DDFA_CHECK_LAUNCH("sample_k_kernel");
  for (int pass = 0; pass < 4; ++pass) {
    radix_hist_kernel<<<grid, kThreads, 0, stream>>>(vuln, num_valid, N, seed, pass, ctl, hist);
    DDFA_CHECK_LAUNCH("radix_hist_kernel");
    radix_pick_kernel<<<1, kBins, 0, stream>>>(pass, ctl, hist);
    DDFA_CHECK_LAUNCH("radix_pick_kernel");
  }
  sample_block_count_kernel<<<nb, kThreads, 0, stream>>>(vuln, num_valid, N, seed, ctl, blk);
  DDFA_CHECK_LAUNCH("sample_block_count_kernel");
  sample_block_scan_kernel<<<1, kThreads, 0, stream>>>(nb, ctl, blk, num_rows, nullptr, 0);
  DDFA_CHECK_LAUNCH("sample_block_scan_kernel");
  sample_write_kernel<<<nb, kThreads, 0, stream>>>(vuln, num_valid, N, seed, ctl, blk, rows);
  DDFA_CHECK_LAUNCH("sample_write_kernel");
  return DDFA_OK;
}

// ---- several ranks: the draw of the global batch in phases, with the exchanges between them left to the caller ----------------
size_t ddfa_node_dp_exchange_words(int32_t world) {
  using namespace ddfa::node;
  if (world < 1) return 0;
  return (size_t)kBins + 3 * (size_t)world;
}

namespace {
int dp_check(const char *who, int32_t N, int32_t rank, int32_t world, const void *workspace, size_t workspace_bytes, const void *exchange) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && world >= 1 && rank >= 0 && rank < world, "%s: num_nodes=%d rank=%d world=%d", who, N, rank, world);
  DDFA_REQUIRE(workspace && exchange, "%s: NULL workspace or exchange buffer", who);
  if (workspace_bytes < ddfa_node_sample_workspace_bytes(N)) {
    set_error("%s: workspace too small (%zu < %zu)", who, workspace_bytes, ddfa_node_sample_workspace_bytes(N));
    return DDFA_ERR_WORKSPACE;
  }
  return DDFA_OK;
}
}  // namespace

int ddfa_node_dp_count(const int32_t *vuln, const int32_t *num_valid, int32_t N, double factor, int32_t rank, int32_t world,
                       int32_t *rows, int32_t *num_rows, void *workspace, size_t workspace_bytes, int32_t *exchange, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  if (int rc = dp_check("ddfa_node_dp_count", N, rank, world, workspace, workspace_bytes, exchange)) return rc;
  DDFA_REQUIRE(num_valid && num_rows && (vuln || N == 0) && (rows || N == 0), "ddfa_node_dp_count: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  int32_t *ctl = static_cast<int32_t *>(workspace);
  const int32_t nb = num_blocks(N) > 0 ? num_blocks(N) : 1;
  DDFA_CUDA(cudaMemsetAsync(ctl, 0, sizeof(int32_t) * (kCtl + kBins), stream));
  DDFA_CUDA(cudaMemsetAsync(exchange, 0, sizeof(int32_t) * ddfa_node_dp_exchange_words(world), stream));
  sample_count_kernel<<<(unsigned)min(nb, 4 * kNumSMs), kThreads, 0, stream>>>(vuln, num_valid, N, exchange + kBins + 2 * rank);
  DDFA_CHECK_LAUNCH("sample_count_kernel");
  if (!(factor >= 0.0)) {       // no undersampling: the rows are every local valid node now
    sample_all_kernel<<<cdiv(N > 0 ? N : 1, kThreads), kThreads, 0, stream>>>(num_valid, N, rows, num_rows);
    DDFA_CHECK_LAUNCH("sample_all_kernel");
  }
  return DDFA_OK;
}

int ddfa_node_dp_plan(int32_t N, double factor, int32_t rank, int32_t world, int64_t *draw, int32_t *status, int32_t *num_rows_global,
                      int32_t *node_offset, void *workspace, size_t workspace_bytes, const int32_t *exchange, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  if (int rc = dp_check("ddfa_node_dp_plan", N, rank, world, workspace, workspace_bytes, exchange)) return rc;
  DDFA_REQUIRE(num_rows_global && node_offset && (!(factor >= 0.0) || (draw && status)), "ddfa_node_dp_plan: NULL pointer");
  dp_plan_kernel<<<1, 1, 0, as_stream(stream_)>>>(exchange + kBins, rank, world, factor, draw, status, static_cast<int32_t *>(workspace),
                                                  num_rows_global, node_offset);
  DDFA_CHECK_LAUNCH("dp_plan_kernel");
  return DDFA_OK;
}

int ddfa_node_dp_radix_hist(const int32_t *vuln, const int32_t *num_valid, int32_t N, uint64_t seed, int32_t pass, void *workspace,
                            size_t workspace_bytes, int32_t *exchange, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  if (int rc = dp_check("ddfa_node_dp_radix_hist", N, 0, 1, workspace, workspace_bytes, exchange)) return rc;
  DDFA_REQUIRE(pass >= 0 && pass < 4, "ddfa_node_dp_radix_hist: pass=%d not in [0, 4)", pass);
  DDFA_REQUIRE(num_valid && (vuln || N == 0), "ddfa_node_dp_radix_hist: NULL pointer");
  const int32_t nb = num_blocks(N) > 0 ? num_blocks(N) : 1;
  radix_hist_kernel<<<(unsigned)min(nb, 4 * kNumSMs), kThreads, 0, as_stream(stream_)>>>(vuln, num_valid, N, seed, pass,
                                                                                          static_cast<int32_t *>(workspace),
                                                                                          reinterpret_cast<uint32_t *>(exchange));
  DDFA_CHECK_LAUNCH("radix_hist_kernel");
  return DDFA_OK;
}

int ddfa_node_dp_radix_pick(int32_t N, int32_t pass, void *workspace, size_t workspace_bytes, int32_t *exchange, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  if (int rc = dp_check("ddfa_node_dp_radix_pick", N, 0, 1, workspace, workspace_bytes, exchange)) return rc;
  DDFA_REQUIRE(pass >= 0 && pass < 4, "ddfa_node_dp_radix_pick: pass=%d not in [0, 4)", pass);
  radix_pick_kernel<<<1, kBins, 0, as_stream(stream_)>>>(pass, static_cast<int32_t *>(workspace), reinterpret_cast<uint32_t *>(exchange));
  DDFA_CHECK_LAUNCH("radix_pick_kernel");
  return DDFA_OK;
}

int ddfa_node_dp_ties(const int32_t *vuln, const int32_t *num_valid, int32_t N, uint64_t seed, int32_t rank, int32_t world, void *workspace,
                      size_t workspace_bytes, int32_t *exchange, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  if (int rc = dp_check("ddfa_node_dp_ties", N, rank, world, workspace, workspace_bytes, exchange)) return rc;
  DDFA_REQUIRE(num_valid && (vuln || N == 0), "ddfa_node_dp_ties: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  int32_t *ctl = static_cast<int32_t *>(workspace);
  int32_t *blk = ctl + kCtl + kBins;
  const int32_t nb = num_blocks(N) > 0 ? num_blocks(N) : 1;
  sample_block_count_kernel<<<nb, kThreads, 0, stream>>>(vuln, num_valid, N, seed, ctl, blk);
  DDFA_CHECK_LAUNCH("sample_block_count_kernel");
  tie_total_kernel<<<1, kThreads, 0, stream>>>(nb, blk, exchange + kBins + 2 * world + rank);
  DDFA_CHECK_LAUNCH("tie_total_kernel");
  return DDFA_OK;
}

int ddfa_node_dp_rows(const int32_t *vuln, const int32_t *num_valid, int32_t N, uint64_t seed, int32_t rank, int32_t world, int32_t *rows,
                      int32_t *num_rows, void *workspace, size_t workspace_bytes, const int32_t *exchange, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  if (int rc = dp_check("ddfa_node_dp_rows", N, rank, world, workspace, workspace_bytes, exchange)) return rc;
  DDFA_REQUIRE(num_valid && num_rows && (vuln || N == 0) && (rows || N == 0), "ddfa_node_dp_rows: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  int32_t *ctl = static_cast<int32_t *>(workspace);
  int32_t *blk = ctl + kCtl + kBins;
  const int32_t nb = num_blocks(N) > 0 ? num_blocks(N) : 1;
  sample_block_scan_kernel<<<1, kThreads, 0, stream>>>(nb, ctl, blk, num_rows, exchange + kBins + 2 * world, rank);
  DDFA_CHECK_LAUNCH("sample_block_scan_kernel");
  sample_write_kernel<<<nb, kThreads, 0, stream>>>(vuln, num_valid, N, seed, ctl, blk, rows);
  DDFA_CHECK_LAUNCH("sample_write_kernel");
  return DDFA_OK;
}

int ddfa_node_bce_global(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows, const int32_t *num_rows_global,
                         int32_t N, float pos_weight, float grad_scale, float *loss_out, float *dlogits, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  DDFA_REQUIRE(N >= 0, "ddfa_node_bce_global: num_nodes=%d < 0", N);
  DDFA_REQUIRE(logits && vuln && rows && num_rows && num_rows_global, "ddfa_node_bce_global: NULL pointer");
  node_bce_kernel<true><<<1, 1024, 0, as_stream(stream_)>>>(logits, vuln, rows, num_rows, num_rows_global, pos_weight, grad_scale, loss_out,
                                                            dlogits);
  DDFA_CHECK_LAUNCH("node_bce_kernel");
  return DDFA_OK;
}

int ddfa_node_head_fwd(const float *h_final, const float *x, const int32_t *rows, const int32_t *num_rows, int32_t N, int32_t D,
                       const float *const *mlp_w, const float *const *mlp_b, int32_t L, float *mlp_act, float *logits, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  DDFA_REQUIRE(N >= 0 && D > 0 && L >= 1 && L <= kMaxLayers, "ddfa_node_head_fwd: bad shape N=%d D=%d num_layers=%d", N, D, L);
  DDFA_REQUIRE(num_rows && mlp_w && mlp_b, "ddfa_node_head_fwd: NULL pointer");
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(h_final && x && rows && logits && (L == 1 || mlp_act), "ddfa_node_head_fwd: NULL pointer");
  for (int i = 0; i < L; ++i) DDFA_REQUIRE(mlp_w[i] && mlp_b[i], "ddfa_node_head_fwd: MLP layer %d pointer NULL", i);
  cudaStream_t stream = as_stream(stream_);
  const int32_t K = 2 * D;
  const size_t plane = (size_t)N * K;
  for (int i = 0; i + 1 < L; ++i) {
    const dim3 grid(cdiv(N, BM), cdiv(K, BN));
    float *act = mlp_act + (size_t)i * plane;
    if (i == 0)
      head_gemm_kernel<true, true, kBiasRelu><<<grid, 256, 0, stream>>>(nullptr, h_final, x, rows, num_rows, D, K, K, mlp_w[i], mlp_b[i],
                                                                        nullptr, act, nullptr, nullptr);
    else
      head_gemm_kernel<false, true, kBiasRelu><<<grid, 256, 0, stream>>>(mlp_act + (size_t)(i - 1) * plane, nullptr, nullptr, rows, num_rows, D,
                                                                         K, K, mlp_w[i], mlp_b[i], nullptr, act, nullptr, nullptr);
    DDFA_CHECK_LAUNCH("head_gemm_kernel");
  }
  if (L == 1)
    head_out_kernel<true><<<cdiv(N, 8), 256, 0, stream>>>(nullptr, h_final, x, rows, num_rows, D, K, mlp_w[0], mlp_b[0], logits);
  else
    head_out_kernel<false><<<cdiv(N, 8), 256, 0, stream>>>(mlp_act + (size_t)(L - 2) * plane, nullptr, nullptr, rows, num_rows, D, K,
                                                           mlp_w[L - 1], mlp_b[L - 1], logits);
  DDFA_CHECK_LAUNCH("head_out_kernel");
  return DDFA_OK;
}

int ddfa_node_bce(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows, int32_t N, float pos_weight,
                  float *loss_out, float *dlogits, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  DDFA_REQUIRE(N >= 0, "ddfa_node_bce: num_nodes=%d < 0", N);
  DDFA_REQUIRE(logits && vuln && rows && num_rows, "ddfa_node_bce: NULL pointer");
  node_bce_kernel<false><<<1, 1024, 0, as_stream(stream_)>>>(logits, vuln, rows, num_rows, nullptr, pos_weight, 1.f, loss_out, dlogits);
  DDFA_CHECK_LAUNCH("node_bce_kernel");
  return DDFA_OK;
}

int ddfa_node_bce_scaled(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows, int32_t N,
                         float pos_weight, float grad_scale, float *loss_out, float *dlogits, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  DDFA_REQUIRE(N >= 0, "ddfa_node_bce_scaled: num_nodes=%d < 0", N);
  DDFA_REQUIRE(logits && vuln && rows && num_rows, "ddfa_node_bce_scaled: NULL pointer");
  node_bce_kernel<true><<<1, 1024, 0, as_stream(stream_)>>>(logits, vuln, rows, num_rows, nullptr, pos_weight, grad_scale, loss_out,
                                                                 dlogits);
  DDFA_CHECK_LAUNCH("node_bce_kernel");
  return DDFA_OK;
}

size_t ddfa_node_head_bwd_workspace_bytes(int32_t N, int32_t D) {
  using namespace ddfa::node;
  if (N < 0 || D < 0) return 0;
  const size_t K = 2 * (size_t)D;
  return sizeof(float) * (2 * (size_t)N * K + (size_t)kHeadChunks * (K * K + K));
}

int ddfa_node_head_bwd(const float *dlogits, const float *h_final, const float *x, const int32_t *rows, const int32_t *num_rows, int32_t N,
                       int32_t D, const float *const *mlp_w, int32_t L, const float *mlp_act, float *dh_final, float *dx,
                       float *const *dmlp_w, float *const *dmlp_b, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::node;
  DDFA_REQUIRE(N >= 0 && D > 0 && L >= 1 && L <= kMaxLayers, "ddfa_node_head_bwd: bad shape N=%d D=%d num_layers=%d", N, D, L);
  DDFA_REQUIRE(num_rows && mlp_w && dmlp_w && dmlp_b, "ddfa_node_head_bwd: NULL pointer");
  for (int i = 0; i < L; ++i) DDFA_REQUIRE(mlp_w[i] && dmlp_w[i] && dmlp_b[i], "ddfa_node_head_bwd: MLP layer %d pointer NULL", i);
  // dh_final == dx == NULL: the MLP gradients only (the encoder is frozen), no [N, D] plane is written
  DDFA_REQUIRE((dh_final == nullptr) == (dx == nullptr), "ddfa_node_head_bwd: dh_final and dx are both NULL (MLP gradients only) or both given");
  DDFA_REQUIRE(N == 0 || (dlogits && h_final && x && rows && (L == 1 || mlp_act)), "ddfa_node_head_bwd: NULL pointer");
  if (workspace_bytes < ddfa_node_head_bwd_workspace_bytes(N, D) || workspace == nullptr) {
    set_error("ddfa_node_head_bwd: workspace too small (%zu < %zu)", workspace_bytes, ddfa_node_head_bwd_workspace_bytes(N, D));
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t stream = as_stream(stream_);
  const int32_t K = 2 * D;
  const size_t plane = (size_t)N * K;
  float *buf[2] = {static_cast<float *>(workspace), static_cast<float *>(workspace) + plane};
  float *partial = buf[1] + plane;
  const bool input_grads = dh_final != nullptr;
  if (N > 0 && input_grads) {       // both planes whole: zero outside the listed rows
    DDFA_CUDA(cudaMemsetAsync(dh_final, 0, sizeof(float) * (size_t)N * D, stream));
    DDFA_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * (size_t)N * D, stream));
  }
  // last layer: Linear(2D, 1) on in = act[L-2] (or the gathered rows when L == 1)
  const float *in_last = L == 1 ? nullptr : mlp_act + (size_t)(L - 2) * plane;
  int rc = L == 1 ? launch_wgrad<true>(dlogits, nullptr, h_final, x, rows, num_rows, D, 1, dmlp_w[0], dmlp_b[0], partial, stream)
                  : launch_wgrad<false>(dlogits, in_last, nullptr, nullptr, rows, num_rows, D, 1, dmlp_w[L - 1], dmlp_b[L - 1], partial, stream);
  if (rc) return rc;
  if (N == 0 || (L == 1 && !input_grads)) return DDFA_OK;
  const unsigned g_elem = cdiv((int64_t)N * K, 256);
  if (L == 1) {
    head_last_bwd_kernel<true><<<g_elem, 256, 0, stream>>>(dlogits, mlp_w[0], nullptr, rows, num_rows, D, N, nullptr, dh_final, dx);
    DDFA_CHECK_LAUNCH("head_last_bwd_kernel");
    return DDFA_OK;
  }
  head_last_bwd_kernel<false><<<g_elem, 256, 0, stream>>>(dlogits, mlp_w[L - 1], in_last, rows, num_rows, D, N, buf[0], nullptr, nullptr);
  DDFA_CHECK_LAUNCH("head_last_bwd_kernel");
  int cur = 0;
  for (int i = L - 2; i >= 0; --i) {
    const float *dout = buf[cur];
    const float *in = i == 0 ? nullptr : mlp_act + (size_t)(i - 1) * plane;
    rc = i == 0 ? launch_wgrad<true>(dout, nullptr, h_final, x, rows, num_rows, D, K, dmlp_w[0], dmlp_b[0], partial, stream)
                : launch_wgrad<false>(dout, in, nullptr, nullptr, rows, num_rows, D, K, dmlp_w[i], dmlp_b[i], partial, stream);
    if (rc) return rc;
    if (i == 0 && !input_grads) break;
    const dim3 grid(cdiv(N, BM), cdiv(K, BN));
    if (i == 0)
      head_gemm_kernel<false, false, kScatter><<<grid, 256, 0, stream>>>(dout, nullptr, nullptr, rows, num_rows, D, K, K, mlp_w[0], nullptr,
                                                                         nullptr, nullptr, dh_final, dx);
    else
      head_gemm_kernel<false, false, kMask><<<grid, 256, 0, stream>>>(dout, nullptr, nullptr, rows, num_rows, D, K, K, mlp_w[i], nullptr, in,
                                                                      buf[1 - cur], nullptr, nullptr);
    DDFA_CHECK_LAUNCH("head_gemm_kernel");
    cur = 1 - cur;
  }
  return DDFA_OK;
}

}  // extern "C"
