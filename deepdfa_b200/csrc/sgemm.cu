// SIMT engine: generic row-major fp32 GEMM,  C[M,N] = alpha * op(A) op(B) + beta * C.
//
// This is the fp32 FFMA building block of the DDFA_ENGINE_SIMT path (any hidden width) and the
// bisecting reference for the tcgen05 engine.  It stands in for the cuBLAS SGEMM calls behind
// nn.Linear / nn.GRUCell in the reference (ggnn.py:57-60,71-80) and for autograd's wgrad/dgrad.
//
// 128x128x16 CTA tile, 256 threads, 8x8 register tile per thread, double-buffered shared memory
// with register prefetch.  split_k > 1 distributes K over gridDim.z and accumulates with RED.ADD
// (used for the weight gradients, where M,N are tiny and K = number of nodes).
#include "common.cuh"

namespace ddfa {

constexpr int BM = 128, BN = 128, BK = 16, LDS_PAD = 4;

// Loads a [128 (mn) x 16 (k)] tile into registers.  KCONTIG: memory is contiguous along k
// (element (mn,k) at p[mn*ld + k]); otherwise contiguous along mn (element at p[k*ld + mn]).
template <bool KCONTIG>
__device__ __forceinline__ void load_tile(const float *__restrict__ p, int ld, int mn0, int k0, int MN, int Kend,
                                          bool vec_ok, float4 (&reg)[2]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int mn, k;
    if (KCONTIG) { mn = mn0 + (t >> 2) + i * 64; k = k0 + (t & 3) * 4; }
    else         { k = k0 + (t >> 5) + i * 8;    mn = mn0 + (t & 31) * 4; }
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (KCONTIG) {
      if (mn < MN) {
        const float *q = p + (int64_t)mn * ld + k;
        if (vec_ok && k + 3 < Kend) v = *reinterpret_cast<const float4 *>(q);
        else {
          if (k + 0 < Kend) v.x = q[0];
          if (k + 1 < Kend) v.y = q[1];
          if (k + 2 < Kend) v.z = q[2];
          if (k + 3 < Kend) v.w = q[3];
        }
      }
    } else {
      if (k < Kend) {
        const float *q = p + (int64_t)k * ld + mn;
        if (vec_ok && mn + 3 < MN) v = *reinterpret_cast<const float4 *>(q);
        else {
          if (mn + 0 < MN) v.x = q[0];
          if (mn + 1 < MN) v.y = q[1];
          if (mn + 2 < MN) v.z = q[2];
          if (mn + 3 < MN) v.w = q[3];
        }
      }
    }
    reg[i] = v;
  }
}

template <bool KCONTIG>
__device__ __forceinline__ void store_tile(float (*s)[BM + LDS_PAD], const float4 (&reg)[2]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (KCONTIG) {
      const int mn = (t >> 2) + i * 64, k = (t & 3) * 4;
      s[k + 0][mn] = reg[i].x; s[k + 1][mn] = reg[i].y; s[k + 2][mn] = reg[i].z; s[k + 3][mn] = reg[i].w;
    } else {
      const int k = (t >> 5) + i * 8, mn = (t & 31) * 4;
      *reinterpret_cast<float4 *>(&s[k][mn]) = reg[i];
    }
  }
}

// ZSLICE: split-K slice z writes its own [M x ldc] block at C + z * M * ldc (deterministic split-K: the slices are added in z
// order by splitk_reduce_kernel instead of with atomics)
template <bool TA, bool TB, bool ZSLICE = false>
__global__ void __launch_bounds__(256) sgemm_kernel(int M, int N, int K, float alpha, const float *__restrict__ A,
                                                    int lda, const float *__restrict__ B, int ldb, float beta,
                                                    float *__restrict__ C, int ldc, int k_per_split, int use_atomic,
                                                    int vec_a, int vec_b) {
  if constexpr (ZSLICE) C += (int64_t)blockIdx.z * M * ldc;
  __shared__ __align__(16) float As[2][BK][BM + LDS_PAD];
  __shared__ __align__(16) float Bs[2][BK][BN + LDS_PAD];
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  // op(A)[m][k]: !TA -> A[m*lda+k] (k contiguous); TA -> A[k*lda+m] (m contiguous)
  // op(B)[k][n]: !TB -> B[k*ldb+n] (n contiguous); TB -> B[n*ldb+k] (k contiguous)
  if (kbeg < kend) {
    load_tile<!TA>(A, lda, m0, kbeg, M, kend, vec_a, ra);
    load_tile<TB>(B, ldb, n0, kbeg, N, kend, vec_b, rb);
    store_tile<!TA>(As[0], ra);
    store_tile<TB>(Bs[0], rb);
  }
  __syncthreads();
  int buf = 0;
  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    const bool has_next = k0 + BK < kend;
    if (has_next) {
      load_tile<!TA>(A, lda, m0, k0 + BK, M, kend, vec_a, ra);
      load_tile<TB>(B, ldb, n0, k0 + BK, N, kend, vec_b, rb);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (has_next) {
      store_tile<!TA>(As[buf ^ 1], ra);
      store_tile<TB>(Bs[buf ^ 1], rb);
    }
    __syncthreads();
    buf ^= 1;
  }
  if (kbeg >= kend && (use_atomic || blockIdx.z > 0)) return;

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n >= N) continue;
      float *c = C + (int64_t)m * ldc + n;
      const float v = alpha * acc[i][j];
      if (use_atomic) atomicAdd(c, v);
      else *c = (beta == 0.f) ? v : fmaf(beta, *c, v);
    }
  }
}

// Small problems (weight folding, MLP head forward / backward: M, N <= a few hundred) would occupy 1-6 of the 132 SMs with the
// 128x128 tile and run for tens of microseconds; this kernel uses 32x32 output tiles so the same work spreads over dozens of
// CTAs.  64 threads, 4x4 outputs per thread (16 FFMA per two LDS.128 — the 2x2 form of round 1 was bound by its shared-memory
// loads), K staged 32 at a time through shared memory with the next stage prefetched into registers.
// KC: the operand tile [32 (mn) x 32 (k)] is contiguous along k in memory (element (mn, k) at p[mn * ld + k]); else along mn.
template <bool KC>
__device__ __forceinline__ void small_fetch(const float *__restrict__ p, int ld, int mn0, int MN, int k0, int K, bool vec, float4 (&r)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e4 = threadIdx.x + 64 * i;                 // 256 float4 per operand stage
    const int mn = KC ? (e4 >> 3) : 4 * (e4 & 7), k = KC ? 4 * (e4 & 7) : (e4 >> 3);
    const int gmn = mn0 + mn, gk = k0 + k;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (KC) {
      if (gmn < MN) {
        const float *q = p + (int64_t)gmn * ld + gk;
        if (vec && gk + 3 < K) v = *reinterpret_cast<const float4 *>(q);
        else {
          if (gk + 0 < K) v.x = q[0];
          if (gk + 1 < K) v.y = q[1];
          if (gk + 2 < K) v.z = q[2];
          if (gk + 3 < K) v.w = q[3];
        }
      }
    } else if (gk < K) {
      const float *q = p + (int64_t)gk * ld + gmn;
      if (vec && gmn + 3 < MN) v = *reinterpret_cast<const float4 *>(q);
      else {
        if (gmn + 0 < MN) v.x = q[0];
        if (gmn + 1 < MN) v.y = q[1];
        if (gmn + 2 < MN) v.z = q[2];
        if (gmn + 3 < MN) v.w = q[3];
      }
    }
    r[i] = v;
  }
}
template <bool KC>
__device__ __forceinline__ void small_stage(float (*s)[36], const float4 (&r)[4]) {      // s[k][mn]
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e4 = threadIdx.x + 64 * i;
    if (KC) {
      const int mn = e4 >> 3, k = 4 * (e4 & 7);
      s[k + 0][mn] = r[i].x; s[k + 1][mn] = r[i].y; s[k + 2][mn] = r[i].z; s[k + 3][mn] = r[i].w;
    } else {
      *reinterpret_cast<float4 *>(&s[e4 >> 3][4 * (e4 & 7)]) = r[i];
    }
  }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(64) sgemm_small_kernel(int M, int N, int K, float alpha, const float *__restrict__ A, int lda,
                                                         const float *__restrict__ B, int ldb, float beta, float *__restrict__ C,
                                                         int ldc, int vec_a, int vec_b, int k_per_split, int use_atomic) {
  constexpr int KB = 32;
  __shared__ __align__(16) float As[KB][36];      // [k][m]   (row stride 36 floats: 16-byte aligned rows for the LDS.128 below)
  __shared__ __align__(16) float Bs[KB][36];      // [k][n]
  const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  float4 ra[4], rb[4];
  float acc[4][4] = {};
  const int kbeg = blockIdx.z * k_per_split;                   // split-K: gridDim.z slices of K, accumulated with RED.ADD (beta == 1)
  K = min(K, kbeg + k_per_split);
  small_fetch<!TA>(A, lda, m0, M, kbeg, K, vec_a != 0, ra);   // A element (m, k) at A[m*lda + k] (k-contiguous) unless transposed
  small_fetch<TB>(B, ldb, n0, N, kbeg, K, vec_b != 0, rb);    // B element (k, n) at B[k*ldb + n] (n-contiguous) unless transposed
  for (int k0 = kbeg; k0 < K; k0 += KB) {
    small_stage<!TA>(As, ra);
    small_stage<TB>(Bs, rb);
    __syncthreads();
    if (k0 + KB < K) {
      small_fetch<!TA>(A, lda, m0, M, k0 + KB, K, vec_a != 0, ra);
      small_fetch<TB>(B, ldb, n0, N, k0 + KB, K, vec_b != 0, rb);
    }
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      const float4 a = *reinterpret_cast<const float4 *>(&As[k][4 * ty]);
      const float4 b = *reinterpret_cast<const float4 *>(&Bs[k][4 * tx]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + 4 * ty + i, n = n0 + 4 * tx + j;
      if (m < M && n < N) {
        float *c = C + (int64_t)m * ldc + n;
        const float v = alpha * acc[i][j];
        if (use_atomic) atomicAdd(c, v);
        else *c = (beta == 0.f) ? v : fmaf(beta, *c, v);
      }
    }
}

// C[i] += sum over z of part[z][i], z in order (one thread per element of the dense [M x N] C block)
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float *__restrict__ part, int nz, int M, int N, float *__restrict__ C,
                                                            int ldc) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  float s = 0.f;
  for (int z = 0; z < nz; ++z) s += part[(int64_t)z * M * N + i];
  float *c = C + (i / N) * ldc + i % N;
  *c += s;
}

int sgemm_splitk_ordered_slices(int K, int split_k) {
  const int k_tiles = (K + BK - 1) / BK;
  if (split_k > k_tiles) split_k = k_tiles > 0 ? k_tiles : 1;
  if (split_k < 1) split_k = 1;
  const int kps = ((k_tiles + split_k - 1) / split_k) * BK;
  return K > 0 ? (K + kps - 1) / kps : 1;
}

int sgemm_splitk_ordered(int M, int N, int K, float alpha, const float *A, int lda, const float *B, int ldb, float *C, int ldc,
                         int split_k, float *part, cudaStream_t stream) {
  if (M == 0 || N == 0 || K == 0) return DDFA_OK;
  const int k_tiles = (K + BK - 1) / BK;
  if (split_k > k_tiles) split_k = k_tiles;
  if (split_k < 1) split_k = 1;
  const int kps = ((k_tiles + split_k - 1) / split_k) * BK;
  const int nz = sgemm_splitk_ordered_slices(K, split_k);
  const int vec_a = aligned16(A) && (lda % 4 == 0), vec_b = aligned16(B) && (ldb % 4 == 0);
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, nz);
  sgemm_kernel<true, false, true><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, 0.f, part, N, kps, 0, vec_a, vec_b);
  DDFA_CHECK_LAUNCH("sgemm_kernel(z slices)");
  const int64_t tot = (int64_t)M * N;
  splitk_reduce_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(part, nz, M, N, C, ldc);
  DDFA_CHECK_LAUNCH("splitk_reduce_kernel");
  return DDFA_OK;
}

int sgemm(int ta, int tb, int M, int N, int K, float alpha, const float *A, int lda, const float *B, int ldb,
          float beta, float *C, int ldc, int split_k, cudaStream_t stream) {
  if (M == 0 || N == 0) return DDFA_OK;
  if (split_k < 1) split_k = 1;
  if (split_k == 1 && (int64_t)M * N <= 512 * 512 && K <= 4096) {
    dim3 grid((N + 31) / 32, (M + 31) / 32);
    // An accumulating product (beta == 1) with a long K and few output tiles — the MLP head's weight gradients, K = batch size —
    // is a chain of K/32 load latencies on a handful of SMs: slice K over gridDim.z and accumulate with RED.ADD instead (not in
    // deterministic mode: each output element is then one CTA's sum over all of K).
    int split = 1;
    const int tiles = (int)(grid.x * grid.y);
    if (beta == 1.f && K >= 256 && tiles < kNumSMs && !deterministic()) {
      split = (2 * kNumSMs + tiles - 1) / tiles;
      if (split > K / 64) split = K / 64;
      if (split < 1) split = 1;
    }
    int kps = ((K + split - 1) / split + 31) / 32 * 32;
    if (kps < 32) kps = 32;
    grid.z = K > kps ? (K + kps - 1) / kps : 1;
    const int atomic = grid.z > 1;
    const int va = aligned16(A) && (lda % 4 == 0), vb = aligned16(B) && (ldb % 4 == 0);
#define LAUNCH_S(TA, TB) sgemm_small_kernel<TA, TB><<<grid, 64, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, va, vb, kps, atomic)
    if (!ta && !tb) LAUNCH_S(false, false);
    else if (!ta && tb) LAUNCH_S(false, true);
    else if (ta && !tb) LAUNCH_S(true, false);
    else LAUNCH_S(true, true);
#undef LAUNCH_S
    DDFA_CHECK_LAUNCH("sgemm_small_kernel");
    return DDFA_OK;
  }
  int k_tiles = (K + BK - 1) / BK;
  if (split_k > k_tiles) split_k = k_tiles > 0 ? k_tiles : 1;
  const int k_per_split = ((k_tiles + split_k - 1) / split_k) * BK;
  const int use_atomic = split_k > 1;
  if (use_atomic && deterministic()) {
    set_error("sgemm: split_k > 1 accumulates with atomics; deterministic mode needs sgemm_splitk_ordered");
    return DDFA_ERR_UNSUPPORTED;
  }
  if (use_atomic && beta != 1.f) {
    set_error("ddfa_sgemm: split_k > 1 requires beta == 1 (atomic accumulation into C)");
    return DDFA_ERR_INVALID_ARG;
  }
  const int vec_a = aligned16(A) && (lda % 4 == 0);
  const int vec_b = aligned16(B) && (ldb % 4 == 0);
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, split_k);
  if (grid.y > 65535u) {
    set_error("ddfa_sgemm: M=%d too large for grid.y", M);
    return DDFA_ERR_UNSUPPORTED;
  }
#define LAUNCH(TA, TB) sgemm_kernel<TA, TB><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, k_per_split, use_atomic, vec_a, vec_b)
  if (!ta && !tb) LAUNCH(false, false);
  else if (!ta && tb) LAUNCH(false, true);
  else if (ta && !tb) LAUNCH(true, false);
  else LAUNCH(true, true);
#undef LAUNCH
  DDFA_CHECK_LAUNCH("sgemm_kernel");
  return DDFA_OK;
}

}  // namespace ddfa

extern "C" int ddfa_sgemm(int trans_a, int trans_b, int32_t m, int32_t n, int32_t k, float alpha, const float *a,
                          int32_t lda, const float *b, int32_t ldb, float beta, float *c, int32_t ldc,
                          int32_t split_k, void *stream) {
  using namespace ddfa;
  DDFA_REQUIRE(m >= 0 && n >= 0 && k >= 0, "ddfa_sgemm: negative dimension");
  DDFA_REQUIRE(split_k <= 1 || !deterministic(),
               "ddfa_sgemm: split_k > 1 has no deterministic form (DDFA_TUNE_DETERMINISTIC = 1): use split_k = 1");
  DDFA_REQUIRE((m == 0 || n == 0) || (a && b && c) || k == 0, "ddfa_sgemm: NULL pointer");
  return sgemm(trans_a, trans_b, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, split_k, as_stream(stream));
}
