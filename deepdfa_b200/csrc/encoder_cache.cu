// Batch assembly from an encoder cache: the rows h_T and x a frozen graph encoder computed once for every node of an arena,
// gathered for a list of graph ids.  A graph's nodes are contiguous in the arena and in the batch, so each graph is one
// contiguous slab of n * D floats per plane, copied with 16-byte vector loads and stores by as many warps as its size needs.
// No CSR is built and no edge is read: the readout, the node head and their backward read graph_ptr and the rows only.
//
// Offsets are 64-bit: at Big-Vul size (~10^7 nodes) a plane passes 2^32 bytes, and at D = 512 it passes 2^31 elements.
#include "common.cuh"

namespace ddfa {

constexpr int kCacheChunkVec = 128;         // float4 per chunk and plane: one warp, four float4 per lane (2 KB per plane)
constexpr int kCacheCopyThreads = 256;      // 8 warps per CTA, each taking chunks in a grid-stride loop
constexpr int kCacheMaxCtas = kNumSMs * 8;

// ws layout: int32 err, int32 node_ptr[B + 1], int32 chunk_ptr[B + 1].  A graph of n nodes is ceil(n * D / 4 / kCacheChunkVec)
// chunks (none when it has no node), so a graph gets as many warps' worth of work as its size needs.  The scan writes only the
// workspace; the outputs (graph_ptr included) are written by the copy kernel, which runs only when err == 0: a bad id or a node
// total that disagrees with batch_nodes leaves them untouched.
__global__ void __launch_bounds__(1024) cache_scan_kernel(const int32_t *__restrict__ ids, int32_t B, int32_t G,
                                                          const int32_t *__restrict__ node_off, int32_t n_all, int32_t D,
                                                          int32_t n_expect, int32_t *__restrict__ node_ptr,
                                                          int32_t *__restrict__ chunk_ptr, int32_t *__restrict__ err) {
  __shared__ int32_t sn[32], sc[32];
  __shared__ int32_t carry_n, carry_c;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { carry_n = 0; carry_c = 0; }
  __syncthreads();
  for (int base = 0; base < B; base += 1024) {
    const int b = base + (int)threadIdx.x;
    int32_t n = 0, c = 0;
    if (b < B) {
      const int32_t id = ids[b];
      if (id < 0 || id >= G) atomicAdd(err, 1);
      else {
        const int32_t n0 = node_off[id], n1 = node_off[id + 1];
        if (n0 < 0 || n1 < n0 || n1 > n_all) atomicAdd(err, 1);   // node_off of another arena than the cache's planes
        else {
          n = n1 - n0;
          c = (int32_t)(((int64_t)n * (D >> 2) + kCacheChunkVec - 1) / kCacheChunkVec);
        }
      }
    }
    int32_t xn = n, xc = c;              // block-wide inclusive scan of (n, c)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t yn = __shfl_up_sync(0xffffffffu, xn, o), yc = __shfl_up_sync(0xffffffffu, xc, o);
      if (lane >= o) { xn += yn; xc += yc; }
    }
    if (lane == 31) { sn[warp] = xn; sc[warp] = xc; }
    __syncthreads();
    if (warp == 0) {
      int32_t wn = sn[lane], wc = sc[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t yn = __shfl_up_sync(0xffffffffu, wn, o), yc = __shfl_up_sync(0xffffffffu, wc, o);
        if (lane >= o) { wn += yn; wc += yc; }
      }
      sn[lane] = wn; sc[lane] = wc;
    }
    __syncthreads();
    if (b < B) {                         // exclusive prefixes
      node_ptr[b] = carry_n + (warp ? sn[warp - 1] : 0) + xn - n;
      chunk_ptr[b] = carry_c + (warp ? sc[warp - 1] : 0) + xc - c;
    }
    __syncthreads();
    if (threadIdx.x == 1023) { carry_n += sn[31]; carry_c += sc[31]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    node_ptr[B] = carry_n;
    chunk_ptr[B] = carry_c;
    if (carry_n != n_expect) atomicAdd(err, 1 << 16);      // host-side total disagrees with the arena
  }
}

// Each warp takes chunks c = warp id, + total warps, ...: the graph b owning c (binary search of chunk_ptr), then float4
// [(c - chunk_ptr[b]) * kCacheChunkVec, + kCacheChunkVec) of graph b's slab in both planes (lane-interleaved, coalesced).  The lane
// holding a row's first float4 copies that row's _VULN word.  graph_ptr is written by a grid-stride loop over the graphs.
__global__ void __launch_bounds__(kCacheCopyThreads) cache_copy_kernel(const int32_t *__restrict__ ids, int32_t B,
                                                                       const int32_t *__restrict__ node_off,
                                                                       const int32_t *__restrict__ vuln_all, const float4 *__restrict__ h_all,
                                                                       const float4 *__restrict__ x_all, int32_t D,
                                                                       const int32_t *__restrict__ node_ptr, const int32_t *__restrict__ chunk_ptr,
                                                                       const int32_t *__restrict__ err, int32_t *__restrict__ out_graph_ptr,
                                                                       int32_t *__restrict__ out_vuln, float4 *__restrict__ out_h,
                                                                       float4 *__restrict__ out_x) {
  if (*err != 0) return;                   // bad id or inconsistent total: leave the outputs alone, the host reports it
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
  for (int b = tid; b <= B; b += nthreads) out_graph_ptr[b] = node_ptr[b];
  const int lane = threadIdx.x & 31;
  const int warp = tid >> 5, nwarps = nthreads >> 5;
  const int32_t total = chunk_ptr[B];
  const int64_t q = (int64_t)(D >> 2);                              // float4 per row
  for (int32_t c = warp; c < total; c += nwarps) {
    int lo = 0, hi = B - 1;                                         // the last b with chunk_ptr[b] <= c (empty graphs skipped)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (chunk_ptr[mid] <= c) lo = mid; else hi = mid - 1;
    }
    const int b = lo;
    const int32_t id = ids[b];
    const int32_t n0 = node_off[id], n = node_off[id + 1] - n0;
    const int32_t o = node_ptr[b];
    const int64_t len = (int64_t)n * q;
    const int64_t first = (int64_t)(c - chunk_ptr[b]) * kCacheChunkVec;
    const float4 *hs = h_all + (int64_t)n0 * q, *xs = x_all + (int64_t)n0 * q;
    float4 *hd = out_h + (int64_t)o * q, *xd = out_x + (int64_t)o * q;
#pragma unroll
    for (int k = 0; k < kCacheChunkVec / 32; ++k) {
      const int64_t i = first + k * 32 + lane;
      if (i < len) {
        const float4 a = __ldg(hs + i), v = __ldg(xs + i);
        hd[i] = a;
        xd[i] = v;
        if (i % q == 0) out_vuln[o + i / q] = vuln_all[n0 + i / q];
      }
    }
  }
}

}  // namespace ddfa

extern "C" {

size_t ddfa_cache_batch_workspace_bytes(int32_t batch_size) { return sizeof(int32_t) * (2 * (size_t)(batch_size < 0 ? 0 : batch_size) + 3); }

int ddfa_cache_batch(const int32_t *graph_ids, int32_t batch_size, int32_t num_graphs, const int32_t *node_off, const int32_t *vuln_all,
                     const float *h_all, const float *x_all, int32_t num_nodes_all, int32_t D, int32_t batch_nodes, int32_t *out_graph_ptr,
                     int32_t *out_vuln, float *out_h, float *out_x, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(batch_size > 0 && num_graphs > 0 && num_nodes_all >= 0 && batch_nodes >= 0 && D > 0 && D % 4 == 0,
               "ddfa_cache_batch: bad sizes (B=%d G=%d N_all=%d N=%d D=%d; D must be a positive multiple of 4)", batch_size, num_graphs,
               num_nodes_all, batch_nodes, D);
  DDFA_REQUIRE(graph_ids && node_off && out_graph_ptr, "ddfa_cache_batch: NULL pointer");
  DDFA_REQUIRE(num_nodes_all == 0 || (vuln_all && h_all && x_all), "ddfa_cache_batch: NULL cache plane");
  DDFA_REQUIRE(batch_nodes == 0 || (out_vuln && out_h && out_x), "ddfa_cache_batch: NULL output rows");
  DDFA_REQUIRE(aligned16(h_all) && aligned16(x_all) && aligned16(out_h) && aligned16(out_x),
               "ddfa_cache_batch: h_all, x_all, out_h and out_x need 16-byte alignment (rows are copied as float4)");
  // chunk counts are int32: a batch's row planes stay below 2^31 chunks of 2 KB (4 TB)
  if (workspace == nullptr || workspace_bytes < ddfa_cache_batch_workspace_bytes(batch_size)) {
    set_error("ddfa_cache_batch: workspace too small (%zu < %zu)", workspace_bytes, ddfa_cache_batch_workspace_bytes(batch_size));
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t stream = as_stream(stream_);
  int32_t *err = static_cast<int32_t *>(workspace);
  int32_t *node_ptr = err + 1;
  int32_t *chunk_ptr = node_ptr + batch_size + 1;
  DDFA_CUDA(cudaMemsetAsync(err, 0, sizeof(int32_t), stream));
  cache_scan_kernel<<<1, 1024, 0, stream>>>(graph_ids, batch_size, num_graphs, node_off, num_nodes_all, D, batch_nodes, node_ptr,
                                            chunk_ptr, err);
  DDFA_CHECK_LAUNCH("cache_scan_kernel");
  // enough warps for every chunk when the total is small (at most one chunk more per graph than the rows need), at most
  // kCacheMaxCtas CTAs striding over a large one
  const int64_t chunks = ((int64_t)batch_nodes * (D / 4) + kCacheChunkVec - 1) / kCacheChunkVec + batch_size;
  const int64_t want = (chunks + kCacheCopyThreads / 32 - 1) / (kCacheCopyThreads / 32);
  const int ctas = (int)(want < kCacheMaxCtas ? want : kCacheMaxCtas);
  cache_copy_kernel<<<ctas, kCacheCopyThreads, 0, stream>>>(graph_ids, batch_size, node_off, vuln_all, reinterpret_cast<const float4 *>(h_all),
                                                            reinterpret_cast<const float4 *>(x_all), D, node_ptr, chunk_ptr, err, out_graph_ptr,
                                                            out_vuln, reinterpret_cast<float4 *>(out_h), reinterpret_cast<float4 *>(out_x));
  DDFA_CHECK_LAUNCH("cache_copy_kernel");
  return DDFA_OK;
}

}  // extern "C"
