// K5-K7 — concat (never materialised) + GlobalAttentionPooling + MLP head, forward and backward.
// Reference: torch.cat([ggnn_out, feat_embed]) ggnn.py:98; dgl GlobalAttentionPooling(Linear(2D,1))
// ggnn.py:66-68,102 (gate -> softmax_nodes -> sum_nodes(feat*gate)); output_layer ggnn.py:70-80,107.
//
// Forward: one CTA per graph.  Each warp streams node rows o_n = [h_T[n] | x[n]] (coalesced
// 128-bit loads), computes the gate logit with a warp reduction and keeps an ONLINE softmax
// (running max / sum / weighted accumulator), so every node row is read exactly once; the 8
// warp states are merged through shared memory; the MLP then runs in the same CTA on the pooled
// vector (warp per output row, coalesced weight reads).  HBM-bound: 2*N*D*4 bytes read.
#include <math.h>

#include "common.cuh"

namespace ddfa {

constexpr int kMaxChunks = 4;  // D <= 512 in the fused readout (2D <= 1024 floats per node row)
constexpr int kReadoutWarps = 8;
constexpr int kMaxMlpLayers = 16;

// Device pointers of the MLP parameters, passed BY VALUE in kernel-parameter space (the C ABI
// receives host arrays of device pointers; no device-side table needs to be allocated).
struct MlpPtrs {
  const float *w[kMaxMlpLayers];
  const float *b[kMaxMlpLayers];
};

// lane owns chunks c = lane + 32*i (i < CH) of the h half and the same chunks of the x half.
template <int CH>
struct RowFrag {
  float4 v[2][CH];
};

template <int CH>
__device__ __forceinline__ void load_row(RowFrag<CH> &f, const float *__restrict__ h, const float *__restrict__ x,
                                         int64_t n, int D, int lane) {
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int col = (lane + 32 * i) * 4;
    if (col < D) {
      f.v[0][i] = ldg_nc_f4(h + n * D + col);
      f.v[1][i] = ldg_nc_f4(x + n * D + col);
    } else {
      f.v[0][i] = make_float4(0.f, 0.f, 0.f, 0.f);
      f.v[1][i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}
template <int CH>
__device__ __forceinline__ float dot_row(const RowFrag<CH> &a, const RowFrag<CH> &b) {
  float s = 0.f;
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int i = 0; i < CH; ++i) s += f4_dot(a.v[p][i], b.v[p][i]);
  return s;
}

template <int CH>
__global__ void __launch_bounds__(kReadoutWarps * 32) readout_mlp_fwd_kernel(
    const float *__restrict__ h, const float *__restrict__ x, const int32_t *__restrict__ graph_ptr, int32_t D,
    const float *__restrict__ w_gate, const float *__restrict__ b_gate, const MlpPtrs mlp, int32_t L,
    float *__restrict__ pooled, float *__restrict__ logits,
    float *__restrict__ gate_logit, float *__restrict__ seg_max, float *__restrict__ seg_sum,
    float *__restrict__ mlp_act, int32_t B) {
  extern __shared__ __align__(16) float sm[];
  const int D2 = 2 * D;
  float *s_acc = sm;                             // [warps][2D]
  float *s_m = s_acc + kReadoutWarps * D2;       // [warps]
  float *s_l = s_m + kReadoutWarps;              // [warps]
  float *s_in = s_l + kReadoutWarps;             // [2D]  MLP ping
  float *s_out = s_in + D2;                      // [2D]  MLP pong
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];

  RowFrag<CH> wg;
  load_row<CH>(wg, w_gate, w_gate + D, 0, D, lane);  // w_gate = [w_h | w_x], both of length D
  const float bg = b_gate[0];

  float m = -INFINITY, l = 0.f;
  RowFrag<CH> acc;
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int i = 0; i < CH; ++i) acc.v[p][i] = make_float4(0.f, 0.f, 0.f, 0.f);

  // U node rows per iteration: their loads and warp reductions are independent (memory-level parallelism; the
  // one-row-at-a-time version was a chain of ~1 us global-load latencies), one online-softmax update for the group.
  constexpr int U = (CH == 1) ? 4 : (CH == 2 ? 2 : 1);
  for (int32_t nb = n0 + warp; nb < n1; nb += kReadoutWarps * U) {
    RowFrag<CH> o[U];
    float g[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int32_t n = nb + u * kReadoutWarps;
      if (n < n1) load_row<CH>(o[u], h, x, n, D, lane);
      else {
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int i = 0; i < CH; ++i) o[u].v[q][i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) g[u] = dot_row<CH>(o[u], wg);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
      for (int u = 0; u < U; ++u) g[u] += __shfl_xor_sync(0xffffffffu, g[u], off);
    float m_new = m;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int32_t n = nb + u * kReadoutWarps;
      g[u] = (n < n1) ? g[u] + bg : -INFINITY;
      if (n < n1 && gate_logit && lane == 0) gate_logit[n] = g[u];
      m_new = fmaxf(m_new, g[u]);
    }
    // first iteration: exp(-inf) = 0 (m_new is finite when the gate logits are).  A NaN logit (skipped by fmaxf) has p = NaN, a +inf
    // one p = exp(inf - inf) = NaN; the NaN reaches l and acc and, through fmaf(NaN, 0, .), the merge below even from a warp whose
    // max stayed -inf: the graph pools to NaN, as in torch's softmax.  A -inf logit differs: torch gives its row weight 0, but a
    // warp whose first group holds only -inf logits takes p = exp(-inf + inf) = NaN here and the graph pools to NaN.  With finite
    // gate weights and bias a logit is -inf only when its row is not finite, and then torch's sum (0 * inf) is NaN as well
    const float scale = expf(m - m_new);
    float p[U];
#pragma unroll
    for (int u = 0; u < U; ++u) p[u] = expf(g[u] - m_new);   // exp(-inf) = 0 for rows past the graph
    float psum = 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u) psum += p[u];
    l = fmaf(l, scale, psum);
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        float4 &a = acc.v[q][i];
        a.x *= scale; a.y *= scale; a.z *= scale; a.w *= scale;
#pragma unroll
        for (int u = 0; u < U; ++u) f4_fma(a, p[u], o[u].v[q][i]);
      }
    m = m_new;
  }
  // publish warp state
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int col = (lane + 32 * i) * 4;
      if (col < D) *reinterpret_cast<float4 *>(&s_acc[warp * D2 + q * D + col]) = acc.v[q][i];
    }
  if (lane == 0) { s_m[warp] = m; s_l[warp] = l; }
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < kReadoutWarps; ++w) M = fmaxf(M, s_m[w]);
  float Lsum = 0.f;
  float wscale[kReadoutWarps];
#pragma unroll
  for (int w = 0; w < kReadoutWarps; ++w) {
    wscale[w] = (s_m[w] == -INFINITY) ? 0.f : expf(s_m[w] - M);
    Lsum = fmaf(s_l[w], wscale[w], Lsum);
  }
  const float inv = Lsum > 0.f ? 1.f / Lsum : 0.f;  // empty graph -> pooled = 0 (sum over no nodes)
  for (int j = threadIdx.x; j < D2; j += blockDim.x) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kReadoutWarps; ++w) v = fmaf(s_acc[w * D2 + j], wscale[w], v);
    v *= inv;
    s_in[j] = v;
    pooled[(int64_t)b * D2 + j] = v;
  }
  if (threadIdx.x == 0) {
    if (seg_max) seg_max[b] = M;
    if (seg_sum) seg_sum[b] = Lsum;
  }
  if (L <= 0) return;
  __syncthreads();
  // MLP: (L-1) x [Linear(2D,2D) + ReLU], then Linear(2D,1)
  for (int layer = 0; layer < L; ++layer) {
    const float *W = mlp.w[layer];
    const float *bias = mlp.b[layer];
    const int rows = (layer == L - 1) ? 1 : D2;
    // R output rows per warp iteration: their weight loads are independent (a row at a time was a chain of L2 latencies,
    // 2D / 8 of them per warp and layer); per row the same lane partition and shuffle tree as before, so the sums are unchanged
    constexpr int R = 4;
    for (int r0 = warp * R; r0 < rows; r0 += kReadoutWarps * R) {
      float sacc[R];
#pragma unroll
      for (int j = 0; j < R; ++j) sacc[j] = 0.f;
      for (int k = lane * 4; k < D2; k += 128) {
        const float4 iv = *reinterpret_cast<const float4 *>(&s_in[k]);
        float4 wv[R];
#pragma unroll
        for (int j = 0; j < R; ++j)
          wv[j] = (r0 + j < rows) ? ldg_nc_f4(W + (int64_t)(r0 + j) * D2 + k) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < R; ++j) sacc[j] += f4_dot(wv[j], iv);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int j = 0; j < R; ++j) sacc[j] += __shfl_xor_sync(0xffffffffu, sacc[j], off);
      float mine = sacc[0];
#pragma unroll
      for (int j = 1; j < R; ++j) mine = (lane == j) ? sacc[j] : mine;
      const int r = r0 + lane;
      if (lane < R && r < rows) {
        float y = mine + bias[r];
        if (layer == L - 1) {
          logits[b] = y;
        } else {
          y = relu_nan(y);
          s_out[r] = y;
          if (mlp_act) mlp_act[((int64_t)layer * B + b) * D2 + r] = y;
        }
      }
    }
    __syncthreads();
    float *tmp = s_in; s_in = s_out; s_out = tmp;
  }
}

// ---- readout backward: one CTA per graph --------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(kReadoutWarps * 32) readout_bwd_kernel(
    const float *__restrict__ dpooled, const float *__restrict__ pooled, const float *__restrict__ h,
    const float *__restrict__ x, const int32_t *__restrict__ graph_ptr, int32_t D, const float *__restrict__ w_gate,
    const float *__restrict__ gate_logit, const float *__restrict__ seg_max, const float *__restrict__ seg_sum,
    float *__restrict__ dh, float *__restrict__ dx, float *__restrict__ dw_gate, float *__restrict__ db_gate,
    float *__restrict__ partial) {
  // partial == NULL: the graph's dw_gate / db_gate terms are added with atomics; else they go to row b of partial [B][2D] and to
  // partial[B * 2D + b], and the caller sums the rows in graph order (deterministic mode)
  extern __shared__ __align__(16) float sm[];
  const int D2 = 2 * D;
  float *s_dw = sm;  // [warps][2D]
  __shared__ float s_db[kReadoutWarps];
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
  RowFrag<CH> wg, dp, pp;
  load_row<CH>(wg, w_gate, w_gate + D, 0, D, lane);
  load_row<CH>(dp, dpooled + (int64_t)b * D2, dpooled + (int64_t)b * D2 + D, 0, D, lane);
  load_row<CH>(pp, pooled + (int64_t)b * D2, pooled + (int64_t)b * D2 + D, 0, D, lane);
  const float cdot = warp_sum(dot_row<CH>(dp, pp));
  const float M = seg_max[b];
  const float Ls = seg_sum[b];
  const float inv = Ls > 0.f ? 1.f / Ls : 0.f;
  RowFrag<CH> dw;
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int i = 0; i < CH; ++i) dw.v[p][i] = make_float4(0.f, 0.f, 0.f, 0.f);
  float dbg = 0.f;
  for (int32_t n = n0 + warp; n < n1; n += kReadoutWarps) {
    RowFrag<CH> o;
    load_row<CH>(o, h, x, n, D, lane);
    const float alpha = expf(gate_logit[n] - M) * inv;
    const float sdot = warp_sum(dot_row<CH>(o, dp));
    const float dg = alpha * (sdot - cdot);
    dbg += dg;
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        const int col = (lane + 32 * i) * 4;
        if (col < D) {
          const float4 &dpv = dp.v[q][i], &wv = wg.v[q][i], &ov = o.v[q][i];
          if (dh) {          // NULL: the gate-only form (frozen encoder), no [N, D] plane is written
            float4 d;
            d.x = fmaf(alpha, dpv.x, dg * wv.x); d.y = fmaf(alpha, dpv.y, dg * wv.y);
            d.z = fmaf(alpha, dpv.z, dg * wv.z); d.w = fmaf(alpha, dpv.w, dg * wv.w);
            float *dst = (q == 0 ? dh : dx) + (int64_t)n * D + col;
            *reinterpret_cast<float4 *>(dst) = d;
          }
          f4_fma(dw.v[q][i], dg, ov);
        }
      }
  }
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int col = (lane + 32 * i) * 4;
      if (col < D) *reinterpret_cast<float4 *>(&s_dw[warp * D2 + q * D + col]) = dw.v[q][i];
    }
  if (lane == 0) s_db[warp] = dbg;
  __syncthreads();
  for (int j = threadIdx.x; j < D2; j += blockDim.x) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kReadoutWarps; ++w) v += s_dw[w * D2 + j];
    if (partial) partial[(int64_t)b * D2 + j] = v;
    else atomicAdd(dw_gate + j, v);
  }
  if (threadIdx.x == 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kReadoutWarps; ++w) v += s_db[w];
    if (partial) partial[(int64_t)gridDim.x * D2 + b] = v;
    else atomicAdd(db_gate, v);
  }
}

// ---- small helpers for the MLP backward ---------------------------------------------------
// out[m,n] = mask[m,n] <= 0 ? 0 : in[m,n]  (a NaN activation passes its gradient, as in torch)
__global__ void relu_mask_kernel(const float *in, const float *__restrict__ mask, int64_t total, float *out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < total) out[i] = relu_grad(mask[i], in[i]);
}
// DeepLift's rescale rule at a hidden ReLU (captum's `nonlinear`): with z = zg + bias and z' = zrg + bias the pre-activations of the
// input and the reference pass, din *= (relu(z) - relu(z')) / (z - z'), or the plain derivative [act > 0] where |z - z'| < 1e-10
__global__ void __launch_bounds__(256) rescale_relu_kernel(float *__restrict__ din, const float *__restrict__ zg, const float *__restrict__ zrg,
                                                           const float *__restrict__ bias, const float *__restrict__ act, int64_t total,
                                                           int32_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float b = bias[i % n];
  const float z = zg[i] + b, zr = zrg[i] + b;
  const float dz = z - zr;
  din[i] = fabsf(dz) < 1e-10f ? relu_grad(act[i], din[i]) : din[i] * (relu_nan(z) - relu_nan(zr)) / dz;
}
// ---- MLP head over the whole batch (large training batches): hidden layers as one GEMM each + this epilogue, last layer below ----
// a[m, n] = relu(a[m, n] + bias[n]), 4 columns per thread (n % 4 == 0)
__global__ void __launch_bounds__(256) bias_relu_kernel(float *__restrict__ a, const float *__restrict__ bias, int64_t total4, int32_t n4) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= total4) return;
  float4 v = *reinterpret_cast<const float4 *>(a + 4 * i);
  const float4 b = *reinterpret_cast<const float4 *>(bias + 4 * (i % n4));
  v.x = relu_nan(v.x + b.x); v.y = relu_nan(v.y + b.y); v.z = relu_nan(v.z + b.z); v.w = relu_nan(v.w + b.w);
  *reinterpret_cast<float4 *>(a + 4 * i) = v;
}
// logits[b] = in[b, :] . w + bias[0]: one warp per graph, the lane partition and shuffle tree of the in-CTA last layer (same sums)
__global__ void __launch_bounds__(256) mlp_out_kernel(const float *__restrict__ in, const float *__restrict__ w, const float *__restrict__ bias,
                                                      int32_t B, int32_t D2, float *__restrict__ logits) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  float s = 0.f;
  for (int k = lane * 4; k < D2; k += 128) s += f4_dot(ldg_nc_f4(w + k), *reinterpret_cast<const float4 *>(in + (int64_t)b * D2 + k));
  s = warp_sum(s);
  if (lane == 0) logits[b] = s + bias[0];
}

// out[n] += sum_m X[m,n]   (one thread per column, coalesced across threads)
// block = (32 columns) x (8 row partitions); gridDim.y slices the rows (a single row slice owns its columns: plain +=; several
// slices — long M, e.g. the MLP head's bias gradients over a batch of 1024 — accumulate with RED.ADD, except in deterministic mode)
__global__ void __launch_bounds__(256) colsum_accum_kernel(const float *__restrict__ X, int32_t M, int32_t N, float *__restrict__ out) {
  __shared__ float red[8][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  const int rows_per = (M + gridDim.y - 1) / gridDim.y;
  const int m0 = blockIdx.y * rows_per, m1 = min(M, m0 + rows_per);
  float s = 0.f;
  if (n < N)
    for (int m = m0 + threadIdx.y; m < m1; m += 8) s += X[(int64_t)m * N + n];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += red[y][threadIdx.x];
    if (gridDim.y > 1) atomicAdd(out + n, t);
    else out[n] += t;
  }
}

}  // namespace ddfa

extern "C" {

int ddfa_readout_mlp_fwd(const float *h_final, const float *x, const int32_t *graph_ptr, int32_t B, int32_t D,
                         const float *w_gate, const float *b_gate, const float *const *mlp_w, const float *const *mlp_b,
                         int32_t L, float *pooled, float *logits, float *gate_logit, float *seg_max, float *seg_sum,
                         float *mlp_act, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(B >= 0 && D > 0 && D % 4 == 0 && D <= 128 * kMaxChunks, "ddfa_readout_mlp_fwd: unsupported shape B=%d D=%d (D%%4==0, D<=%d)", B, D, 128 * kMaxChunks);
  DDFA_REQUIRE(L >= 0 && L <= kMaxMlpLayers, "ddfa_readout_mlp_fwd: num_layers=%d out of range [0,%d]", L, kMaxMlpLayers);
  if (B == 0) return DDFA_OK;
  DDFA_REQUIRE(h_final && x && graph_ptr && w_gate && b_gate && pooled, "ddfa_readout_mlp_fwd: NULL pointer");
  DDFA_REQUIRE(L == 0 || (mlp_w && mlp_b && logits), "ddfa_readout_mlp_fwd: MLP pointers missing");
  DDFA_REQUIRE(aligned16(h_final) && aligned16(x) && aligned16(w_gate), "ddfa_readout_mlp_fwd: 16-byte alignment required");
  MlpPtrs mp;
  for (int i = 0; i < kMaxMlpLayers; ++i) {
    mp.w[i] = i < L ? mlp_w[i] : nullptr;
    mp.b[i] = i < L ? mlp_b[i] : nullptr;
    if (i < L) DDFA_REQUIRE(mp.w[i] && mp.b[i] && aligned16(mp.w[i]), "ddfa_readout_mlp_fwd: MLP layer %d pointer NULL or unaligned", i);
  }
  cudaStream_t stream = as_stream(stream_);
  const int D2 = 2 * D;
  const size_t smem = sizeof(float) * ((size_t)kReadoutWarps * D2 + 2 * kReadoutWarps + 2 * D2);
  const int ch = (D / 4 + 31) / 32;
  // Large training batches: the in-CTA MLP re-reads every weight matrix (2D x 2D floats from L2) once per graph and is a chain of
  // 2D / 32 load latencies per warp and layer (profiles/r03q: 69 us at B = 1024, ~20 us of it pooling).  With B >= 256 and a place
  // for the hidden activations (mlp_act: training) the kernel only pools, each hidden layer is ONE GEMM over the batch
  // (sgemm_small_kernel) + bias / ReLU, and the last layer a warp per graph.  Same values up to fp32 summation order in the
  // hidden layers; rows are independent of the batch they are in either way.
  bool batched = L >= 1 && B >= 256 && (L == 1 || mlp_act != nullptr) && D2 % 4 == 0 && aligned16(pooled) && aligned16(mlp_act);
  for (int i = 0; i + 1 < L; ++i) batched = batched && aligned16(mp.b[i]);
  const int L_in_kernel = batched ? 0 : L;
#define LAUNCH(CH)                                                                                              \
  readout_mlp_fwd_kernel<CH><<<B, kReadoutWarps * 32, smem, stream>>>(h_final, x, graph_ptr, D, w_gate, b_gate, mp, L_in_kernel, pooled, \
                                                                      logits, gate_logit, seg_max, seg_sum, mlp_act, B)
  if (ch == 1) LAUNCH(1);
  else if (ch == 2) LAUNCH(2);
  else LAUNCH(4);
#undef LAUNCH
  DDFA_CHECK_LAUNCH("readout_mlp_fwd_kernel");
  if (batched) {
    const float *in = pooled;
    for (int i = 0; i + 1 < L; ++i) {
      float *act = mlp_act + (size_t)i * B * D2;
      const int rc = sgemm(0, 1, B, D2, D2, 1.f, in, D2, mp.w[i], D2, 0.f, act, D2, 1, stream);     // act = in @ W_i^T
      if (rc) return rc;
      const int64_t total4 = (int64_t)B * D2 / 4;
      bias_relu_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, stream>>>(act, mp.b[i], total4, D2 / 4);
      DDFA_CHECK_LAUNCH("bias_relu_kernel");
      in = act;
    }
    mlp_out_kernel<<<(B + 7) / 8, 256, 0, stream>>>(in, mp.w[L - 1], mp.b[L - 1], B, D2, logits);
    DDFA_CHECK_LAUNCH("mlp_out_kernel");
  }
  return DDFA_OK;
}

int ddfa_mlp_bwd(const float *dlogits, const float *pooled, const float *mlp_act, const float *const *mlp_w, int32_t B,
                 int32_t D, int32_t L, float *dpooled, float *const *dmlp_w, float *const *dmlp_b, float *scratch,
                 void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(B >= 0 && D > 0 && L >= 1 && L <= kMaxMlpLayers, "ddfa_mlp_bwd: bad shape B=%d D=%d L=%d", B, D, L);
  if (B == 0) return DDFA_OK;
  DDFA_REQUIRE(dlogits && pooled && mlp_w && dpooled && dmlp_w && dmlp_b && scratch, "ddfa_mlp_bwd: NULL pointer");
  DDFA_REQUIRE(L == 1 || mlp_act, "ddfa_mlp_bwd: mlp_act required for num_layers > 1");
  cudaStream_t stream = as_stream(stream_);
  const int D2 = 2 * D;
  float *buf0 = scratch, *buf1 = scratch + (size_t)B * D2;
  // dOut of the current layer: [B, out]; starts as dlogits [B,1]
  const float *dout = dlogits;
  int out_dim = 1;
  for (int i = L - 1; i >= 0; --i) {
    const float *in = (i == 0) ? pooled : mlp_act + (size_t)(i - 1) * B * D2;
    // dW_i[out,2D] += dOut^T[out,B] @ in[B,2D]
    int rc = sgemm(1, 0, out_dim, D2, B, 1.f, dout, out_dim, in, D2, 1.f, dmlp_w[i], D2, 1, stream);
    if (rc) return rc;
    colsum_accum_kernel<<<dim3((out_dim + 31) / 32, B >= 256 && !deterministic() ? (B + 63) / 64 : 1), dim3(32, 8), 0, stream>>>(dout, B, out_dim, dmlp_b[i]);
    DDFA_CHECK_LAUNCH("colsum_accum_kernel");
    // dIn[B,2D] = dOut[B,out] @ W_i[out,2D]
    float *din = (i == 0) ? dpooled : (dout == buf0 ? buf1 : buf0);
    rc = sgemm(0, 0, B, D2, out_dim, 1.f, dout, out_dim, mlp_w[i], D2, 0.f, din, D2, 1, stream);
    if (rc) return rc;
    if (i > 0) {
      const int64_t tot = (int64_t)B * D2;
      relu_mask_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(din, in, tot, din);  // in place
      DDFA_CHECK_LAUNCH("relu_mask_kernel");
      dout = din;
      out_dim = D2;
    }
  }
  return DDFA_OK;
}

int ddfa_mlp_dgrad_rescale(const float *dlogits, const float *pooled, const float *mlp_act, const float *pooled_ref,
                           const float *mlp_act_ref, const float *const *mlp_w, const float *const *mlp_b, int32_t B, int32_t D,
                           int32_t L, float *dpooled, float *scratch, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(B >= 0 && D > 0 && L >= 1 && L <= kMaxMlpLayers, "ddfa_mlp_dgrad_rescale: bad shape B=%d D=%d L=%d", B, D, L);
  if (B == 0) return DDFA_OK;
  DDFA_REQUIRE(dlogits && pooled && pooled_ref && mlp_w && dpooled && scratch, "ddfa_mlp_dgrad_rescale: NULL pointer");
  DDFA_REQUIRE(L == 1 || (mlp_act && mlp_act_ref && mlp_b), "ddfa_mlp_dgrad_rescale: mlp_act, mlp_act_ref and mlp_b required for num_layers > 1");
  cudaStream_t stream = as_stream(stream_);
  const int D2 = 2 * D;
  const size_t plane = (size_t)B * D2;
  float *buf0 = scratch, *buf1 = scratch + plane, *z = scratch + 2 * plane, *zr = scratch + 3 * plane;
  const float *dout = dlogits;
  int out_dim = 1;
  for (int i = L - 1; i >= 0; --i) {
    // dIn[B,2D] = dOut[B,out] @ W_i[out,2D]: the call of ddfa_mlp_bwd
    float *din = (i == 0) ? dpooled : (dout == buf0 ? buf1 : buf0);
    int rc = sgemm(0, 0, B, D2, out_dim, 1.f, dout, out_dim, mlp_w[i], D2, 0.f, din, D2, 1, stream);
    if (rc) return rc;
    if (i == 0) break;
    // in_i = relu(z_{i-1}): the pre-activations of both passes, recomputed from the inputs of layer i - 1 (the forward's hidden-layer
    // GEMM when the batch ran the batched head)
    const float *in = (i == 1) ? pooled : mlp_act + (size_t)(i - 2) * plane;
    const float *in_ref = (i == 1) ? pooled_ref : mlp_act_ref + (size_t)(i - 2) * plane;
    rc = sgemm(0, 1, B, D2, D2, 1.f, in, D2, mlp_w[i - 1], D2, 0.f, z, D2, 1, stream);
    if (rc) return rc;
    rc = sgemm(0, 1, B, D2, D2, 1.f, in_ref, D2, mlp_w[i - 1], D2, 0.f, zr, D2, 1, stream);
    if (rc) return rc;
    const int64_t tot = (int64_t)plane;
    rescale_relu_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(din, z, zr, mlp_b[i - 1], mlp_act + (size_t)(i - 1) * plane,
                                                                           tot, D2);
    DDFA_CHECK_LAUNCH("rescale_relu_kernel");
    dout = din;
    out_dim = D2;
  }
  return DDFA_OK;
}

size_t ddfa_readout_bwd_workspace_bytes(int32_t B, int32_t D) {
  if (B < 0 || D < 0) return 0;
  return sizeof(float) * (size_t)B * (2 * (size_t)D + 1);
}

static int readout_bwd_impl(const char *who, const float *dpooled, const float *pooled, const float *h_final, const float *x,
                            const int32_t *graph_ptr, int32_t B, int32_t D, const float *w_gate, const float *gate_logit,
                            const float *seg_max, const float *seg_sum, float *dh_final, float *dx, float *dw_gate,
                            float *db_gate, void *workspace, size_t workspace_bytes, bool has_ws, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(B >= 0 && D > 0 && D % 4 == 0 && D <= 128 * kMaxChunks, "%s: unsupported shape B=%d D=%d", who, B, D);
  DDFA_REQUIRE(has_ws || !deterministic(),
               "ddfa_readout_bwd has no deterministic form (DDFA_TUNE_DETERMINISTIC = 1): use ddfa_readout_bwd_ws");
  if (B == 0) return DDFA_OK;
  // the _ws form takes dh_final == dx == NULL: only dw_gate / db_gate are computed (the encoder below the readout is frozen)
  DDFA_REQUIRE((dh_final == nullptr) == (dx == nullptr), "%s: dh_final and dx are both NULL (gate gradients only) or both given", who);
  DDFA_REQUIRE(has_ws || dh_final, "%s: dh_final / dx NULL: the gate-only form is ddfa_readout_bwd_ws", who);
  DDFA_REQUIRE(dpooled && pooled && h_final && x && graph_ptr && w_gate && gate_logit && seg_max && seg_sum && dw_gate && db_gate,
               "%s: NULL pointer", who);
  // the kernel reads and writes every [., D] row with 16-byte vector accesses (dh_final / dx may be NULL: aligned16(NULL) holds)
  DDFA_REQUIRE(aligned16(dpooled) && aligned16(pooled) && aligned16(h_final) && aligned16(x) && aligned16(w_gate) && aligned16(dh_final) &&
                   aligned16(dx),
               "%s: 16-byte alignment required", who);
  float *partial = nullptr;
  if (deterministic()) {
    if (workspace == nullptr || workspace_bytes < ddfa_readout_bwd_workspace_bytes(B, D)) {
      set_error("%s: workspace too small (%zu < %zu)", who, workspace_bytes, ddfa_readout_bwd_workspace_bytes(B, D));
      return DDFA_ERR_WORKSPACE;
    }
    partial = static_cast<float *>(workspace);
  }
  cudaStream_t stream = as_stream(stream_);
  const size_t smem = sizeof(float) * (size_t)kReadoutWarps * 2 * D;
  const int ch = (D / 4 + 31) / 32;
#define LAUNCH(CH)                                                                                                    \
  readout_bwd_kernel<CH><<<B, kReadoutWarps * 32, smem, stream>>>(dpooled, pooled, h_final, x, graph_ptr, D, w_gate, gate_logit, \
                                                                  seg_max, seg_sum, dh_final, dx, dw_gate, db_gate, partial)
  if (ch == 1) LAUNCH(1);
  else if (ch == 2) LAUNCH(2);
  else LAUNCH(4);
#undef LAUNCH
  DDFA_CHECK_LAUNCH("readout_bwd_kernel");
  if (partial) {      // the graphs' terms, added in graph order
    colsum_accum_kernel<<<dim3((2 * D + 31) / 32, 1), dim3(32, 8), 0, stream>>>(partial, B, 2 * D, dw_gate);
    DDFA_CHECK_LAUNCH("colsum_accum_kernel");
    colsum_accum_kernel<<<dim3(1, 1), dim3(32, 8), 0, stream>>>(partial + (size_t)B * 2 * D, B, 1, db_gate);
    DDFA_CHECK_LAUNCH("colsum_accum_kernel");
  }
  return DDFA_OK;
}

int ddfa_readout_bwd(const float *dpooled, const float *pooled, const float *h_final, const float *x,
                     const int32_t *graph_ptr, int32_t B, int32_t D, const float *w_gate, const float *gate_logit,
                     const float *seg_max, const float *seg_sum, float *dh_final, float *dx, float *dw_gate,
                     float *db_gate, void *stream_) {
  return readout_bwd_impl("ddfa_readout_bwd", dpooled, pooled, h_final, x, graph_ptr, B, D, w_gate, gate_logit, seg_max, seg_sum,
                          dh_final, dx, dw_gate, db_gate, nullptr, 0, false, stream_);
}

int ddfa_readout_bwd_ws(const float *dpooled, const float *pooled, const float *h_final, const float *x,
                        const int32_t *graph_ptr, int32_t B, int32_t D, const float *w_gate, const float *gate_logit,
                        const float *seg_max, const float *seg_sum, float *dh_final, float *dx, float *dw_gate,
                        float *db_gate, void *workspace, size_t workspace_bytes, void *stream_) {
  return readout_bwd_impl("ddfa_readout_bwd_ws", dpooled, pooled, h_final, x, graph_ptr, B, D, w_gate, gate_logit, seg_max, seg_sum,
                          dh_final, dx, dw_gate, db_gate, workspace, workspace_bytes, true, stream_);
}

}  // extern "C"
