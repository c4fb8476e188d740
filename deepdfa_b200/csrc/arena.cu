// Batch producer (SURVEY.md §8 row f1): assemble a training batch ON THE DEVICE from a resident arena of graphs.
//
// The reference assembles every batch on the host — `dgl.batch([...])` in the GraphDataLoader collate
// (DDFA/sastvd/linevd/datamodule.py:116-141) or on the fly in `BigVulDatasetLineVD.get_indices`
// (DDFA/sastvd/linevd/dataset.py:63-76: `dgl.batch([self[i] ...]).to(device)`) — and DGL then builds CSR lazily on the
// device.  Here the whole dataset lives in HBM once, already in the layout the kernels read (CSR by destination + CSR of
// the transposed graph over ALL graphs, node features, labels; the graphs are disjoint and their nodes contiguous), and a
// batch is a list of graph ids: two small kernels rebase the selected graphs' slices to the batch's node / edge numbering.
// Neighbour lists keep their order (sorted by source id — a constant is subtracted and added), so the result is
// bit-identical to ddfa_build_csr on the collated COO of the same graphs.
#include "common.cuh"

namespace ddfa {

constexpr int kArenaMaxFeats = 8;
struct ArenaFeats {                     // device pointers, passed by value
  const int64_t *in[kArenaMaxFeats];
  int64_t *out[kArenaMaxFeats];
};

// ws layout: int32 edge_ptr[B + 1], int32 err, int32 node_ptr[B + 1].  The scan writes only the workspace: whether an id was bad
// or the totals disagree is known after its last pass, so the outputs (graph_ptr included) are written by the assembler, which
// runs only when err == 0.
__global__ void __launch_bounds__(1024) arena_scan_kernel(const int32_t *__restrict__ ids, int32_t B, int32_t G,
                                                          const int32_t *__restrict__ node_off, const int32_t *__restrict__ indptr,
                                                          int32_t n_expect, int32_t e_expect, int32_t *__restrict__ node_ptr,
                                                          int32_t *__restrict__ edge_ptr, int32_t *__restrict__ err) {
  __shared__ int32_t sn[32], se[32];
  __shared__ int32_t carry_n, carry_e;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { carry_n = 0; carry_e = 0; }
  __syncthreads();
  for (int base = 0; base < B; base += 1024) {
    const int b = base + (int)threadIdx.x;
    int32_t n = 0, e = 0;
    if (b < B) {
      const int32_t id = ids[b];
      if (id < 0 || id >= G) atomicAdd(err, 1);
      else {
        const int32_t n0 = node_off[id], n1 = node_off[id + 1];
        n = n1 - n0;
        e = indptr[n1] - indptr[n0];
      }
    }
    // block-wide inclusive scan of (n, e)
    int32_t xn = n, xe = e;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t yn = __shfl_up_sync(0xffffffffu, xn, o), ye = __shfl_up_sync(0xffffffffu, xe, o);
      if (lane >= o) { xn += yn; xe += ye; }
    }
    if (lane == 31) { sn[warp] = xn; se[warp] = xe; }
    __syncthreads();
    if (warp == 0) {
      int32_t wn = sn[lane], we = se[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t yn = __shfl_up_sync(0xffffffffu, wn, o), ye = __shfl_up_sync(0xffffffffu, we, o);
        if (lane >= o) { wn += yn; we += ye; }
      }
      sn[lane] = wn; se[lane] = we;
    }
    __syncthreads();
    const int32_t pn = carry_n + (warp ? sn[warp - 1] : 0) + xn - n;     // exclusive prefix
    const int32_t pe = carry_e + (warp ? se[warp - 1] : 0) + xe - e;
    if (b < B) { node_ptr[b] = pn; edge_ptr[b] = pe; }
    __syncthreads();
    if (threadIdx.x == 1023) { carry_n += sn[31]; carry_e += se[31]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    node_ptr[B] = carry_n;
    edge_ptr[B] = carry_e;
    if (carry_n != n_expect || carry_e != e_expect) atomicAdd(err, 1 << 16);   // host-side totals disagree with the arena
  }
}

__global__ void __launch_bounds__(128) arena_assemble_kernel(const int32_t *__restrict__ ids, int32_t G, const int32_t *__restrict__ node_off,
                                                             const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                             const int32_t *__restrict__ indptr_t, const int32_t *__restrict__ indices_t,
                                                             const ArenaFeats feats, int32_t K,
                                                             const int32_t *__restrict__ vuln, const int32_t *__restrict__ node_ptr,
                                                             const int32_t *__restrict__ edge_ptr, const int32_t *__restrict__ err,
                                                             int32_t *__restrict__ out_graph_ptr, int32_t *__restrict__ out_indptr,
                                                             int32_t *__restrict__ out_indices, int32_t *__restrict__ out_indptr_t,
                                                             int32_t *__restrict__ out_indices_t, int32_t *__restrict__ out_vuln) {
  if (*err != 0) return;                      // bad id or inconsistent totals: leave the outputs alone, the host reports it
  const int b = blockIdx.x;
  const int32_t id = ids[b];
  const int32_t n0 = node_off[id], n = node_off[id + 1] - n0;
  const int32_t e0 = indptr[n0], e0t = indptr_t[n0], ne = indptr[n0 + n] - e0;
  const int32_t o = node_ptr[b], eo = edge_ptr[b];
  if (threadIdx.x == 0) out_graph_ptr[b] = o;
  if (b == (int)gridDim.x - 1 && threadIdx.x == 0) {   // the sentinels: graph_ptr[B] = N, indptr[N] = indptr_t[N] = E
    const int32_t N = node_ptr[b + 1], E = edge_ptr[b + 1];
    out_graph_ptr[b + 1] = N;
    out_indptr[N] = E;
    out_indptr_t[N] = E;
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    out_indptr[o + i] = indptr[n0 + i] - e0 + eo;
    out_indptr_t[o + i] = indptr_t[n0 + i] - e0t + eo;
    out_vuln[o + i] = vuln[n0 + i];
#pragma unroll
    for (int k = 0; k < kArenaMaxFeats; ++k)
      if (k < K) feats.out[k][o + i] = feats.in[k][n0 + i];
  }
  const int32_t shift = o - n0;
  for (int j = threadIdx.x; j < ne; j += blockDim.x) {
    out_indices[eo + j] = indices[e0 + j] + shift;
    out_indices_t[eo + j] = indices_t[e0t + j] + shift;
  }
}

}  // namespace ddfa

extern "C" {

size_t ddfa_arena_batch_workspace_bytes(int32_t batch_size) { return sizeof(int32_t) * (2 * (size_t)(batch_size < 0 ? 0 : batch_size) + 3); }

int ddfa_arena_batch(const int32_t *graph_ids, int32_t batch_size, int32_t num_graphs, const int32_t *node_off, const int32_t *indptr,
                     const int32_t *indices, const int32_t *indptr_t, const int32_t *indices_t, const int64_t *const *feats,
                     int32_t num_feats, const int32_t *vuln, int32_t batch_nodes, int32_t batch_edges, int32_t *out_graph_ptr,
                     int32_t *out_indptr, int32_t *out_indices, int32_t *out_indptr_t, int32_t *out_indices_t,
                     int64_t *const *out_feats, int32_t *out_vuln, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(batch_size > 0 && num_graphs > 0 && num_feats >= 0 && num_feats <= kArenaMaxFeats && batch_nodes >= 0 && batch_edges >= 0,
               "ddfa_arena_batch: bad sizes (B=%d G=%d K=%d N=%d E=%d)", batch_size, num_graphs, num_feats, batch_nodes, batch_edges);
  DDFA_REQUIRE(graph_ids && node_off && indptr && indices && indptr_t && indices_t && vuln && out_graph_ptr && out_indptr && out_indices &&
                   out_indptr_t && out_indices_t && out_vuln && (num_feats == 0 || (feats && out_feats)),
               "ddfa_arena_batch: NULL pointer");
  ArenaFeats fp = {};
  for (int k = 0; k < num_feats; ++k) {
    DDFA_REQUIRE(feats[k] && out_feats[k], "ddfa_arena_batch: NULL feature array %d", k);
    fp.in[k] = feats[k];
    fp.out[k] = out_feats[k];
  }
  if (workspace == nullptr || workspace_bytes < ddfa_arena_batch_workspace_bytes(batch_size)) {
    set_error("ddfa_arena_batch: workspace too small (%zu < %zu)", workspace_bytes, ddfa_arena_batch_workspace_bytes(batch_size));
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t stream = as_stream(stream_);
  int32_t *edge_ptr = static_cast<int32_t *>(workspace);
  int32_t *err = edge_ptr + batch_size + 1;
  int32_t *node_ptr = err + 1;
  DDFA_CUDA(cudaMemsetAsync(err, 0, sizeof(int32_t), stream));
  arena_scan_kernel<<<1, 1024, 0, stream>>>(graph_ids, batch_size, num_graphs, node_off, indptr, batch_nodes, batch_edges, node_ptr, edge_ptr,
                                            err);
  DDFA_CHECK_LAUNCH("arena_scan_kernel");
  arena_assemble_kernel<<<batch_size, 128, 0, stream>>>(graph_ids, num_graphs, node_off, indptr, indices, indptr_t, indices_t, fp, num_feats,
                                                        vuln, node_ptr, edge_ptr, err, out_graph_ptr, out_indptr, out_indices, out_indptr_t,
                                                        out_indices_t, out_vuln);
  DDFA_CHECK_LAUNCH("arena_assemble_kernel");
  return DDFA_OK;
}

}  // extern "C"
