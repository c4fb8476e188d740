// Statement-level localisation: per-node scores of a batch and IVDetect's top-k statement metric over them, accumulated on the
// device (include/ddfa_b200.h, K9').
//
// Reference: DDFA/sastvd/helpers/evaluate.py:262-322 (eval_statements / eval_statements_inter / eval_statements_list).  Each function
// sorts its statements by score with Python's stable sort (reverse=True keeps node order among equal scores) and asks whether one
// of the first k is vulnerable.  That only depends on `rank`, the number of statements ahead of the first-ranked vulnerable one:
// the vulnerable node of maximum score (lowest node id among equal scores), and ahead of it every node of higher score or of
// equal score and lower id.  top-k is hit iff rank < k, also for functions of fewer than k statements.
//
// Order: one CTA per function (grid-stride over a grid that depends on num_graphs only), two passes over the function's nodes:
// the (score, id) maximum over the vulnerable nodes, then the count ahead of it.  Both are exact (a lexicographic maximum and an
// integer count), every state word is an integer count, per-CTA partials are integers and a one-thread launch adds them in CTA
// order: the state does not depend on scheduling.
#include <math.h>

#include "common.cuh"

namespace ddfa {
namespace stmt {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCtas = 2 * kNumSMs;
constexpr int kTopK = 10;
// state words (DDFA_STMT_STATE_WORDS)
enum { kFunctions = 0, kVulnFunctions = 1, kHit1 = 2, kRankSum = 12, kClean = 13, kNaN = 14, kBatches = 15, kWords = 16 };
constexpr int kFields = 15;         // per-CTA partial: words [0, 15)

// (score, id) ordering of the ranking: a ranks ahead of b
__device__ __forceinline__ bool ahead(float sa, int32_t ia, float sb, int32_t ib) { return sa > sb || (sa == sb && ia < ib); }

__device__ __forceinline__ void best_merge(float &s, int32_t &i, float so, int32_t io) {
  if (io != INT32_MAX && (i == INT32_MAX || ahead(so, io, s, i))) { s = so; i = io; }
}

__global__ void __launch_bounds__(kThreads) stmt_metric_kernel(const float *__restrict__ scores, const int32_t *__restrict__ vuln,
                                                               const int32_t *__restrict__ graph_ptr, int32_t num_valid, int full,
                                                               float threshold, unsigned long long *__restrict__ partials) {
  __shared__ float s_best[kWarps];
  __shared__ int32_t s_bid[kWarps];
  __shared__ int s_flags[kWarps];
  __shared__ int32_t s_cnt[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long acc[kFields];
#pragma unroll
  for (int f = 0; f < kFields; ++f) acc[f] = 0ull;
  for (int32_t b = blockIdx.x; b < num_valid; b += gridDim.x) {
    const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
    // pass 1: first-ranked vulnerable node, NaN flag (bit 0), a score above the threshold (bit 1)
    float best = -INFINITY;
    int32_t bid = INT32_MAX;
    int flags = 0;
    for (int32_t n = n0 + threadIdx.x; n < n1; n += kThreads) {
      const float s = scores[n];
      if (isnan(s)) flags |= 1;
      if (s > threshold) flags |= 2;
      if (vuln[n] != 0) best_merge(best, bid, s, n);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float so = __shfl_xor_sync(0xffffffffu, best, o);
      const int32_t io = __shfl_xor_sync(0xffffffffu, bid, o);
      best_merge(best, bid, so, io);
      flags |= __shfl_xor_sync(0xffffffffu, flags, o);
    }
    if (lane == 0) { s_best[warp] = best; s_bid[warp] = bid; s_flags[warp] = flags; }
    __syncthreads();
    best = s_best[0]; bid = s_bid[0]; flags = s_flags[0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) { best_merge(best, bid, s_best[w], s_bid[w]); flags |= s_flags[w]; }
    const bool vulnerable = bid != INT32_MAX;
    // pass 2: the statements ranked ahead of it
    int32_t cnt = 0;
    if (vulnerable && !(flags & 1))
      for (int32_t n = n0 + threadIdx.x; n < n1; n += kThreads) cnt += ahead(scores[n], n, best, bid) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s_cnt[warp] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      int32_t rank = 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) rank += s_cnt[w];
      acc[kFunctions] += 1ull;
      if (flags & 1) {
        acc[kNaN] += 1ull;
      } else if (vulnerable) {
        acc[kVulnFunctions] += 1ull;
        acc[kRankSum] += (unsigned long long)rank;
#pragma unroll
        for (int k = 1; k <= kTopK; ++k) acc[kHit1 + k - 1] += rank < k ? 1ull : 0ull;
      } else if (full && !(flags & 2)) {
        acc[kClean] += 1ull;
      }
    }
    __syncthreads();      // the shared words are rewritten by the next function
  }
  if (threadIdx.x == 0) {     // thread 0 holds the CTA's counts
#pragma unroll
    for (int f = 0; f < kFields; ++f) partials[blockIdx.x * kFields + f] = acc[f];
  }
}

__global__ void stmt_finish_kernel(const unsigned long long *__restrict__ partials, int ctas, double *__restrict__ state) {
  const int f = threadIdx.x;
  if (f >= kFields) return;
  unsigned long long t = 0ull;
  for (int c = 0; c < ctas; ++c) t += partials[c * kFields + f];
  state[f] += (double)t;
  if (f == 0) state[kBatches] += 1.0;
}

// alpha_n = softmax of the gate logits over the function, the expression of readout_bwd_kernel (csrc/readout.cu)
__global__ void __launch_bounds__(kThreads) attention_kernel(const float *__restrict__ gate_logit, const float *__restrict__ seg_max,
                                                             const float *__restrict__ seg_sum, const int32_t *__restrict__ graph_ptr,
                                                             float *__restrict__ alpha) {
  const int32_t b = blockIdx.x;
  const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
  const float M = seg_max[b];
  const float Ls = seg_sum[b];
  const float inv = Ls > 0.f ? 1.f / Ls : 0.f;
  for (int32_t n = n0 + threadIdx.x; n < n1; n += kThreads) alpha[n] = expf(gate_logit[n] - M) * inv;
}

// warp per node: score[n] (+)= w * sum_d f(x, g), g = dh + dx, lanes over d and a fixed shuffle tree
template <int F>
__global__ void __launch_bounds__(256) input_grad_score_kernel(const float *__restrict__ x, const float *__restrict__ dh,
                                                               const float *__restrict__ dx, int32_t N, int32_t D, float w,
                                                               int accumulate, float *__restrict__ score) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= N) return;
  const int64_t row = n * D;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float g = dh[row + d] + dx[row + d];
    s += F == DDFA_STMT_SCORE_ABS ? fabsf(g) : x[row + d] * g;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) score[n] = accumulate ? fmaf(w, s, score[n]) : w * s;
}

__global__ void __launch_bounds__(256) scale_rows_kernel(const float *__restrict__ x, float alpha, int64_t numel, float *__restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < numel; i += (int64_t)gridDim.x * 256) out[i] = alpha * x[i];
}

__global__ void __launch_bounds__(256) node_probability_kernel(const float *__restrict__ logits, const int32_t *__restrict__ num_rows,
                                                               int32_t N, float *__restrict__ scores) {
  const int32_t S = min(max(*num_rows, 0), N);
  for (int32_t n = blockIdx.x * 256 + threadIdx.x; n < N; n += gridDim.x * 256)
    scores[n] = n < S ? 1.f / (1.f + expf(-logits[n])) : 0.f;    // eval_metrics.cu's p: what predictions() stores
}

// ---- DeepLift / DeepLiftShap / GradientShap inputs ----------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11), key = the 64-bit seed, counter (batch, sample, index, column word): all four output words
__device__ __forceinline__ uint4 philox4(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint64_t seed) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return make_uint4(c0, c1, c2, c3);
}

// the column word of the counter: the noise of column quad q is q, the baseline's q | kBaseWord, the function's alpha kAlphaWord
constexpr uint32_t kBaseWord = 0x40000000u, kAlphaWord = 0x80000000u;

__device__ __forceinline__ float uniform24(uint32_t w) { return (float)(w >> 8) * 0x1p-24f; }       // [0, 1), exact

// Box-Muller on the words (a, b): u1 = ((a >> 8) + 1) 2^-24 in (0, 1], u2 = (b >> 8) 2^-24
__device__ __forceinline__ float2 gauss2(uint32_t a, uint32_t b) {
  const float r = sqrtf(-2.f * logf((float)((a >> 8) + 1u) * 0x1p-24f));
  float s, c;
  sincospif(2.f * uniform24(b), &s, &c);
  return make_float2(r * c, r * s);
}

__device__ __forceinline__ float4 gauss4(uint4 w) {
  const float2 p = gauss2(w.x, w.y), q = gauss2(w.z, w.w);
  return make_float4(p.x, p.y, q.x, q.y);
}

// one CTA per function (grid-stride): alpha_b (given, or drawn from word 0 of the function's counter), then per column quad of its
// nodes x~ = x + noise_stdev eps, b = baseline_stdev eps', diff = x~ - b, input = fmaf(alpha_b, diff, b)
__global__ void __launch_bounds__(256) shap_input_kernel(const float *__restrict__ x, const int32_t *__restrict__ graph_ptr, int32_t B,
                                                        int32_t D, float alpha, float noise_stdev, float base_stdev, uint64_t seed,
                                                        const int64_t *__restrict__ counter, uint32_t sample, float *__restrict__ input,
                                                        float *__restrict__ diff) {
  const uint32_t batch = (uint32_t)(uint64_t)*counter;
  const int32_t quads = D / 4;
  for (int32_t b = blockIdx.x; b < B; b += gridDim.x) {
    const float a = alpha >= 0.f ? alpha : uniform24(philox4(batch, sample, (uint32_t)b, kAlphaWord, seed).x);
    const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
    const int64_t units = (int64_t)(n1 - n0) * quads;
    for (int64_t i = threadIdx.x; i < units; i += 256) {
      const int32_t n = n0 + (int32_t)(i / quads), q = (int32_t)(i % quads);
      const int64_t off = (int64_t)n * D + 4 * q;
      float4 xt = *reinterpret_cast<const float4 *>(x + off);
      float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (noise_stdev > 0.f) {
        const float4 e = gauss4(philox4(batch, sample, (uint32_t)n, (uint32_t)q, seed));
        xt.x += noise_stdev * e.x; xt.y += noise_stdev * e.y; xt.z += noise_stdev * e.z; xt.w += noise_stdev * e.w;
      }
      if (base_stdev > 0.f) {
        const float4 e = gauss4(philox4(batch, sample, (uint32_t)n, (uint32_t)q | kBaseWord, seed));
        bv = make_float4(base_stdev * e.x, base_stdev * e.y, base_stdev * e.z, base_stdev * e.w);
      }
      const float4 d = make_float4(xt.x - bv.x, xt.y - bv.y, xt.z - bv.z, xt.w - bv.w);
      *reinterpret_cast<float4 *>(diff + off) = d;
      *reinterpret_cast<float4 *>(input + off) = make_float4(fmaf(a, d.x, bv.x), fmaf(a, d.y, bv.y), fmaf(a, d.z, bv.z), fmaf(a, d.w, bv.w));
    }
  }
}

inline int grid_for(int64_t units, int per_cta) {
  const int64_t c = (units + per_cta - 1) / per_cta;
  return (int)(c < 1 ? 1 : (c > 8 * kNumSMs ? 8 * kNumSMs : c));
}

}  // namespace stmt
}  // namespace ddfa

extern "C" {

size_t ddfa_stmt_metric_workspace_bytes(void) { return sizeof(unsigned long long) * ddfa::stmt::kFields * ddfa::stmt::kMaxCtas; }

int ddfa_stmt_metric(const float *scores, const int32_t *vuln, const int32_t *graph_ptr, int32_t num_graphs, int32_t num_valid,
                     int32_t mode, float threshold, double *state, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_graphs >= 0 && num_valid >= 0 && num_valid <= num_graphs,
               "ddfa_stmt_metric: need 0 <= num_valid (%d) <= num_graphs (%d)", num_valid, num_graphs);
  DDFA_REQUIRE(mode == DDFA_STMT_MODE_VULN_ONLY || mode == DDFA_STMT_MODE_FULL, "ddfa_stmt_metric: mode %d unknown", mode);
  DDFA_REQUIRE(state && workspace, "ddfa_stmt_metric: NULL pointer");
  DDFA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0 && (reinterpret_cast<uintptr_t>(state) & 7u) == 0,
               "ddfa_stmt_metric: state and workspace must be 8-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_stmt_metric_workspace_bytes(), "ddfa_stmt_metric: workspace of %zu bytes, need %zu",
               workspace_bytes, ddfa_stmt_metric_workspace_bytes());
  DDFA_REQUIRE(num_valid == 0 || (scores && vuln && graph_ptr), "ddfa_stmt_metric: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  auto *partials = static_cast<unsigned long long *>(workspace);
  const int ctas = num_graphs < 1 ? 1 : (num_graphs > kMaxCtas ? kMaxCtas : num_graphs);
  stmt_metric_kernel<<<ctas, kThreads, 0, stream>>>(scores, vuln, graph_ptr, num_valid, mode == DDFA_STMT_MODE_FULL, threshold, partials);
  DDFA_CHECK_LAUNCH("stmt_metric_kernel");
  stmt_finish_kernel<<<1, 32, 0, stream>>>(partials, ctas, state);
  DDFA_CHECK_LAUNCH("stmt_finish_kernel");
  return DDFA_OK;
}

int ddfa_stmt_attention(const float *gate_logit, const float *seg_max, const float *seg_sum, const int32_t *graph_ptr,
                        int32_t num_graphs, float *alpha, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_graphs >= 0, "ddfa_stmt_attention: num_graphs=%d < 0", num_graphs);
  if (num_graphs == 0) return DDFA_OK;
  DDFA_REQUIRE(gate_logit && seg_max && seg_sum && graph_ptr && alpha, "ddfa_stmt_attention: NULL pointer");
  attention_kernel<<<num_graphs, kThreads, 0, as_stream(stream_)>>>(gate_logit, seg_max, seg_sum, graph_ptr, alpha);
  DDFA_CHECK_LAUNCH("stmt_attention_kernel");
  return DDFA_OK;
}

int ddfa_stmt_input_grad_score(const float *x, const float *dh, const float *dx, int32_t num_nodes, int32_t dim, int32_t rule,
                               float weight, int32_t accumulate, float *score, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_nodes >= 0 && dim > 0, "ddfa_stmt_input_grad_score: need num_nodes (%d) >= 0 and dim (%d) > 0", num_nodes, dim);
  DDFA_REQUIRE(rule == DDFA_STMT_SCORE_ABS || rule == DDFA_STMT_SCORE_X_TIMES, "ddfa_stmt_input_grad_score: rule %d unknown", rule);
  if (num_nodes == 0) return DDFA_OK;
  DDFA_REQUIRE(dh && dx && score && (x || rule == DDFA_STMT_SCORE_ABS), "ddfa_stmt_input_grad_score: NULL pointer");
  const int grid = (num_nodes + 7) / 8;
  cudaStream_t stream = as_stream(stream_);
  if (rule == DDFA_STMT_SCORE_ABS)
    input_grad_score_kernel<DDFA_STMT_SCORE_ABS><<<grid, 256, 0, stream>>>(x, dh, dx, num_nodes, dim, weight, accumulate, score);
  else
    input_grad_score_kernel<DDFA_STMT_SCORE_X_TIMES><<<grid, 256, 0, stream>>>(x, dh, dx, num_nodes, dim, weight, accumulate, score);
  DDFA_CHECK_LAUNCH("stmt_input_grad_score_kernel");
  return DDFA_OK;
}

int ddfa_stmt_scale_input(const float *x, float alpha, int32_t num_nodes, int32_t dim, float *out, void *image, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_nodes >= 0 && dim > 0, "ddfa_stmt_scale_input: need num_nodes (%d) >= 0 and dim (%d) > 0", num_nodes, dim);
  DDFA_REQUIRE(image == nullptr || dim == 128, "ddfa_stmt_scale_input: activation images exist for dim == 128 only (dim=%d)", dim);
  if (num_nodes == 0) return DDFA_OK;
  DDFA_REQUIRE(x && out && x != out, "ddfa_stmt_scale_input: NULL pointer, or out aliases x");
  const int64_t numel = (int64_t)num_nodes * dim;
  scale_rows_kernel<<<grid_for(numel, 256), 256, 0, as_stream(stream_)>>>(x, alpha, numel, out);
  DDFA_CHECK_LAUNCH("stmt_scale_rows_kernel");
  if (image) return ddfa_act_to_image(out, num_nodes, dim, image, stream_);
  return DDFA_OK;
}

int ddfa_stmt_attribution_score(const float *diff, const float *dh, const float *dx, int32_t num_nodes, int32_t dim, float weight,
                                int32_t accumulate, float *score, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_nodes >= 0 && dim > 0, "ddfa_stmt_attribution_score: need num_nodes (%d) >= 0 and dim (%d) > 0", num_nodes, dim);
  if (num_nodes == 0) return DDFA_OK;
  DDFA_REQUIRE(diff && dh && dx && score, "ddfa_stmt_attribution_score: NULL pointer");
  // the x * g rule of ddfa_stmt_input_grad_score with the difference tensor in place of x: the same sums, bit for bit
  input_grad_score_kernel<DDFA_STMT_SCORE_X_TIMES><<<(num_nodes + 7) / 8, 256, 0, as_stream(stream_)>>>(diff, dh, dx, num_nodes, dim,
                                                                                                     weight, accumulate, score);
  DDFA_CHECK_LAUNCH("stmt_attribution_score_kernel");
  return DDFA_OK;
}

int ddfa_stmt_shap_input(const float *x, const int32_t *graph_ptr, int32_t num_graphs, int32_t num_nodes, int32_t dim, float alpha,
                         float noise_stdev, float baseline_stdev, uint64_t seed, const int64_t *counter, int32_t sample, float *input,
                         float *diff, void *image, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_graphs >= 0 && num_nodes >= 0 && dim > 0 && dim % 4 == 0,
               "ddfa_stmt_shap_input: need num_graphs (%d) >= 0, num_nodes (%d) >= 0 and dim (%d) a positive multiple of 4", num_graphs,
               num_nodes, dim);
  DDFA_REQUIRE(alpha <= 1.f && noise_stdev >= 0.f && baseline_stdev >= 0.f && sample >= 0,
               "ddfa_stmt_shap_input: need alpha <= 1 (negative: drawn), stdevs >= 0 and sample >= 0");
  DDFA_REQUIRE(image == nullptr || dim == 128, "ddfa_stmt_shap_input: activation images exist for dim == 128 only (dim=%d)", dim);
  if (num_nodes == 0 || num_graphs == 0) return DDFA_OK;
  DDFA_REQUIRE(x && graph_ptr && counter && input && diff, "ddfa_stmt_shap_input: NULL pointer");
  DDFA_REQUIRE(x != input && x != diff && input != diff, "ddfa_stmt_shap_input: input, diff and x must not alias");
  DDFA_REQUIRE(aligned16(x) && aligned16(input) && aligned16(diff), "ddfa_stmt_shap_input: 16-byte alignment required");
  shap_input_kernel<<<num_graphs < 8 * kNumSMs ? num_graphs : 8 * kNumSMs, 256, 0, as_stream(stream_)>>>(
      x, graph_ptr, num_graphs, dim, alpha, noise_stdev, baseline_stdev, seed, counter, (uint32_t)sample, input, diff);
  DDFA_CHECK_LAUNCH("stmt_shap_input_kernel");
  if (image) return ddfa_act_to_image(input, num_nodes, dim, image, stream_);
  return DDFA_OK;
}

int ddfa_stmt_node_probability(const float *logits, const int32_t *num_rows, int32_t num_nodes, float *scores, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::stmt;
  DDFA_REQUIRE(num_nodes >= 0, "ddfa_stmt_node_probability: num_nodes=%d < 0", num_nodes);
  if (num_nodes == 0) return DDFA_OK;
  DDFA_REQUIRE(logits && num_rows && scores, "ddfa_stmt_node_probability: NULL pointer");
  node_probability_kernel<<<grid_for(num_nodes, 256), 256, 0, as_stream(stream_)>>>(logits, num_rows, num_nodes, scores);
  DDFA_CHECK_LAUNCH("stmt_node_probability_kernel");
  return DDFA_OK;
}

}  // extern "C"
