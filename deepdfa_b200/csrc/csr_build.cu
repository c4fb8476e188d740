// COO -> CSR (by destination) + CSR of the transposed graph (by source), on the device.
// Replaces what DGL builds lazily inside update_all (reference call site ggnn.py:95); the COO
// arrays are what DGLGraph.edges() / dgl.batch hand over (dataset.py:76).
//
// Pipeline (all on `stream`, no host sync):
//   1. zero counters             2. histogram of dst (and src) with RED.ADD
//   3. exclusive scan -> indptr  4. scatter with atomic cursors into a temp array
//   5. per-slot rank sort inside each row -> neighbour lists sorted by id, so the result (and
//      therefore the fp32 summation order of the gather) is deterministic.
// Out-of-range node ids are dropped and counted in workspace[0] (int32).
#include "common.cuh"

namespace ddfa {

template <typename IdxT>
__global__ void csr_count_kernel(const IdxT *__restrict__ src, const IdxT *__restrict__ dst, int64_t E,
                                 int32_t N, int32_t *__restrict__ indptr, int32_t *__restrict__ indptr_t,
                                 int32_t *__restrict__ err) {
  int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  int64_t s = (int64_t)src[e], d = (int64_t)dst[e];
  if (s < 0 || s >= N || d < 0 || d >= N) {
    atomicAdd(err, 1);
    return;
  }
  if (indptr) atomicAdd(&indptr[d + 1], 1);
  if (indptr_t) atomicAdd(&indptr_t[s + 1], 1);
}

// One CTA scans one array in place: a[1..n] (counts) -> inclusive prefix sums; a[0] stays 0.
// blockIdx.x selects which of the two arrays.  1024 threads x 16 items per pass (all 16 loads in flight) with a carry:
// 38 401 counts = 3 passes (4 items per pass took 10 passes of three barriers and a memory round trip each, ~20 us).
__global__ void __launch_bounds__(1024) csr_scan_kernel(int32_t *a0, int32_t *a1, int32_t n) {
  int32_t *a = blockIdx.x == 0 ? a0 : a1;
  if (a == nullptr) return;
  a += 1;
  constexpr int kItems = 16;
  __shared__ int32_t warp_tot[32];
  __shared__ int32_t carry_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (int32_t base = 0; base < n; base += 1024 * kItems) {
    const int32_t i0 = base + tid * kItems;
    int32_t v[kItems];
#pragma unroll
    for (int j = 0; j < kItems; ++j) v[j] = (i0 + j < n) ? a[i0 + j] : 0;
#pragma unroll
    for (int j = 1; j < kItems; ++j) v[j] += v[j - 1];
    int32_t x = v[kItems - 1];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int32_t t = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int32_t y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      warp_tot[lane] = t;
    }
    __syncthreads();
    const int32_t carry = carry_s;
    const int32_t excl = x - v[kItems - 1] + (wid > 0 ? warp_tot[wid - 1] : 0) + carry;
#pragma unroll
    for (int j = 0; j < kItems; ++j)
      if (i0 + j < n) a[i0 + j] = v[j] + excl;
    __syncthreads();
    if (tid == 1023) carry_s = carry + warp_tot[31];
    __syncthreads();
  }
}

// Multi-CTA scan for large arrays (the single-CTA scan above is a serial chain of passes: 153 600 counts = 10 passes, ~100 us per
// CSR build at C1, paid every step on the host-batch path).  Three short launches, blockIdx.y = which array:
//   csr_block_sum_kernel   sums[y][1 + b] = sum of the b-th block of kScanBlock counts
//   csr_scan_kernel        in-place inclusive scan of sums[y][1 ..]  ->  sums[y][b] = everything before block b
//   csr_block_scan_kernel  in-place inclusive scan of each block of counts + its offset sums[y][b]
constexpr int kScanBlock = 4096;      // 256 threads x 16 items
__global__ void __launch_bounds__(256) csr_block_sum_kernel(const int32_t *a0, const int32_t *a1, int32_t n, int32_t *s0, int32_t *s1) {
  const int32_t *a = blockIdx.y == 0 ? a0 : a1;
  int32_t *sums = blockIdx.y == 0 ? s0 : s1;
  if (a == nullptr) return;
  a += 1;
  const int32_t base = blockIdx.x * kScanBlock;
  int32_t v = 0;
#pragma unroll
  for (int j = 0; j < kScanBlock / 256; ++j) {
    const int32_t i = base + j * 256 + threadIdx.x;      // coalesced
    v += i < n ? a[i] : 0;
  }
  __shared__ int32_t ws[8];
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t t = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += ws[w];
    sums[1 + blockIdx.x] = t;
    if (blockIdx.x == 0) sums[0] = 0;
  }
}
__global__ void __launch_bounds__(256) csr_block_scan_kernel(int32_t *a0, int32_t *a1, int32_t n, const int32_t *s0, const int32_t *s1) {
  int32_t *a = blockIdx.y == 0 ? a0 : a1;
  const int32_t *sums = blockIdx.y == 0 ? s0 : s1;
  if (a == nullptr) return;
  a += 1;
  constexpr int kItems = kScanBlock / 256;
  __shared__ int32_t warp_tot[8];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int32_t i0 = blockIdx.x * kScanBlock + tid * kItems;
  int32_t v[kItems];
#pragma unroll
  for (int j = 0; j < kItems; j += 4) {      // 16-byte loads (a + 1 is 4-byte aligned only: scalar loads, four in a row per sector)
#pragma unroll
    for (int q = 0; q < 4; ++q) v[j + q] = (i0 + j + q < n) ? a[i0 + j + q] : 0;
  }
#pragma unroll
  for (int j = 1; j < kItems; ++j) v[j] += v[j - 1];
  int32_t x = v[kItems - 1];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  int32_t before = sums[blockIdx.x];
#pragma unroll
  for (int w = 0; w < 8; ++w) before += (w < wid) ? warp_tot[w] : 0;
  const int32_t excl = x - v[kItems - 1] + before;
#pragma unroll
  for (int j = 0; j < kItems; ++j)
    if (i0 + j < n) a[i0 + j] = v[j] + excl;
}

template <typename IdxT>
__global__ void csr_fill_kernel(const IdxT *__restrict__ src, const IdxT *__restrict__ dst, int64_t E,
                                int32_t N, const int32_t *__restrict__ indptr,
                                const int32_t *__restrict__ indptr_t, int32_t *__restrict__ cur,
                                int32_t *__restrict__ cur_t, int32_t *__restrict__ tmp,
                                int32_t *__restrict__ tmp_t) {
  int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  int64_t s = (int64_t)src[e], d = (int64_t)dst[e];
  if (s < 0 || s >= N || d < 0 || d >= N) return;
  if (indptr) {
    int32_t p = atomicAdd(&cur[d], 1);
    tmp[indptr[d] + p] = (int32_t)s;
  }
  if (indptr_t) {
    int32_t p = atomicAdd(&cur_t[s], 1);
    tmp_t[indptr_t[s] + p] = (int32_t)d;
  }
}

// One thread per CSR slot: locate the row by binary search, rank the value inside its row.
__global__ void csr_rank_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ tmp,
                                int32_t N, int32_t *__restrict__ indices) {
  const int32_t total = indptr[N];
  int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= total) return;
  int32_t lo = 0, hi = N;  // find row r with indptr[r] <= j < indptr[r+1]
  while (hi - lo > 1) {
    int32_t mid = (lo + hi) >> 1;
    if (indptr[mid] <= j) lo = mid; else hi = mid;
  }
  const int32_t beg = indptr[lo], end = indptr[lo + 1];
  const int32_t val = tmp[j];
  int32_t rank = 0;
  for (int32_t i = beg; i < end; ++i) {
    int32_t w = tmp[i];
    rank += (w < val) || (w == val && i < j);
  }
  indices[beg + rank] = val;
}

__global__ void graph_ptr_kernel(const int64_t *__restrict__ bnn, int32_t B, int32_t *__restrict__ ptr) {
  // single CTA, B is small (<= a few thousand): chunked Hillis-Steele with carry
  __shared__ int32_t buf[1024];
  __shared__ int32_t carry_s;
  if (threadIdx.x == 0) { carry_s = 0; ptr[0] = 0; }
  __syncthreads();
  for (int32_t base = 0; base < B; base += 1024) {
    int32_t i = base + threadIdx.x;
    int32_t v = i < B ? (int32_t)bnn[i] : 0;
    buf[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      int32_t y = threadIdx.x >= o ? buf[threadIdx.x - o] : 0;
      __syncthreads();
      buf[threadIdx.x] += y;
      __syncthreads();
    }
    int32_t carry = carry_s;
    if (i < B) ptr[i + 1] = buf[threadIdx.x] + carry;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + buf[1023];
    __syncthreads();
  }
}

int32_t scan_block_sums_len(int32_t n) { return (n + kScanBlock - 1) / kScanBlock + 1; }

int scan_counts(int32_t *a0, int32_t *a1, int32_t n, int32_t *s0, int32_t *s1, cudaStream_t stream) {
  if (n <= 0) return DDFA_OK;
  const int nb = (n + kScanBlock - 1) / kScanBlock;
  if (n > 4 * kScanBlock && s0 != nullptr && (a1 == nullptr || s1 != nullptr)) {
    csr_block_sum_kernel<<<dim3(nb, 2), 256, 0, stream>>>(a0, a1, n, s0, s1);
    DDFA_CHECK_LAUNCH("csr_block_sum_kernel");
    csr_scan_kernel<<<2, 1024, 0, stream>>>(a0 ? s0 : nullptr, a1 ? s1 : nullptr, nb);
    DDFA_CHECK_LAUNCH("csr_scan_kernel(block sums)");
    csr_block_scan_kernel<<<dim3(nb, 2), 256, 0, stream>>>(a0, a1, n, s0, s1);
    DDFA_CHECK_LAUNCH("csr_block_scan_kernel");
  } else {
    csr_scan_kernel<<<2, 1024, 0, stream>>>(a0, a1, n);
    DDFA_CHECK_LAUNCH("csr_scan_kernel");
  }
  return DDFA_OK;
}

}  // namespace ddfa

extern "C" {

size_t ddfa_build_csr_workspace_bytes(int64_t E, int32_t N) {
  if (E < 0 || N < 0) return 0;
  // [err(4 ints, padded)] [cur N] [cur_t N] [tmp E] [tmp_t E]
  return sizeof(int32_t) * (size_t)(4 + 2 * (size_t)N + 2 * (size_t)E);
}

int ddfa_build_csr(const void *src, const void *dst, int idx_bytes, int64_t E, int32_t N, int32_t *indptr,
                   int32_t *indices, int32_t *indptr_t, int32_t *indices_t, void *workspace,
                   size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(E >= 0 && N >= 0, "ddfa_build_csr: negative size (E=%lld, N=%d)", (long long)E, N);
  DDFA_REQUIRE(E < (int64_t)1 << 31, "ddfa_build_csr: E=%lld exceeds int32 CSR", (long long)E);
  DDFA_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "ddfa_build_csr: idx_bytes must be 4 or 8, got %d", idx_bytes);
  DDFA_REQUIRE((indptr == nullptr) == (indices == nullptr), "ddfa_build_csr: indptr/indices must both be set or both NULL");
  DDFA_REQUIRE((indptr_t == nullptr) == (indices_t == nullptr), "ddfa_build_csr: indptr_t/indices_t must both be set or both NULL");
  DDFA_REQUIRE(E == 0 || (src && dst), "ddfa_build_csr: NULL edge arrays");
  if (workspace_bytes < ddfa_build_csr_workspace_bytes(E, N) || workspace == nullptr) {
    set_error("ddfa_build_csr: workspace too small (%zu < %zu)", workspace_bytes, ddfa_build_csr_workspace_bytes(E, N));
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t stream = as_stream(stream_);
  int32_t *ws = static_cast<int32_t *>(workspace);
  int32_t *err = ws;
  int32_t *cur = ws + 4, *cur_t = cur + N, *tmp = cur_t + N, *tmp_t = tmp + E;
  DDFA_CUDA(cudaMemsetAsync(ws, 0, sizeof(int32_t) * (4 + 2 * (size_t)N), stream));
  if (indptr) DDFA_CUDA(cudaMemsetAsync(indptr, 0, sizeof(int32_t) * ((size_t)N + 1), stream));
  if (indptr_t) DDFA_CUDA(cudaMemsetAsync(indptr_t, 0, sizeof(int32_t) * ((size_t)N + 1), stream));
  if (E > 0) {
    const int threads = 256;
    const unsigned blocks = (unsigned)((E + threads - 1) / threads);
    if (idx_bytes == 8)
      csr_count_kernel<int64_t><<<blocks, threads, 0, stream>>>((const int64_t *)src, (const int64_t *)dst, E, N, indptr, indptr_t, err);
    else
      csr_count_kernel<int32_t><<<blocks, threads, 0, stream>>>((const int32_t *)src, (const int32_t *)dst, E, N, indptr, indptr_t, err);
    DDFA_CHECK_LAUNCH("csr_count_kernel");
  }
  if (N > 0) {
    // block sums live in the (not yet used) tmp / tmp_t regions: 1 + nb ints each
    const bool multi = (int64_t)scan_block_sums_len(N) <= E;
    const int rc = scan_counts(indptr, indptr_t, N, multi ? tmp : nullptr, multi ? tmp_t : nullptr, stream);
    if (rc != DDFA_OK) return rc;
  }
  if (E > 0) {
    const int threads = 256;
    const unsigned blocks = (unsigned)((E + threads - 1) / threads);
    if (idx_bytes == 8)
      csr_fill_kernel<int64_t><<<blocks, threads, 0, stream>>>((const int64_t *)src, (const int64_t *)dst, E, N, indptr, indptr_t, cur, cur_t, tmp, tmp_t);
    else
      csr_fill_kernel<int32_t><<<blocks, threads, 0, stream>>>((const int32_t *)src, (const int32_t *)dst, E, N, indptr, indptr_t, cur, cur_t, tmp, tmp_t);
    DDFA_CHECK_LAUNCH("csr_fill_kernel");
    if (indptr) {
      csr_rank_kernel<<<blocks, threads, 0, stream>>>(indptr, tmp, N, indices);
      DDFA_CHECK_LAUNCH("csr_rank_kernel");
    }
    if (indptr_t) {
      csr_rank_kernel<<<blocks, threads, 0, stream>>>(indptr_t, tmp_t, N, indices_t);
      DDFA_CHECK_LAUNCH("csr_rank_kernel(T)");
    }
  }
  return DDFA_OK;
}

int ddfa_graph_ptr(const int64_t *bnn, int32_t B, int32_t *graph_ptr, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(B >= 0 && graph_ptr != nullptr && (B == 0 || bnn != nullptr), "ddfa_graph_ptr: bad arguments (B=%d)", B);
  graph_ptr_kernel<<<1, 1024, 0, as_stream(stream_)>>>(bnn, B, graph_ptr);
  DDFA_CHECK_LAUNCH("graph_ptr_kernel");
  return DDFA_OK;
}

}  // extern "C"
