// Prediction store: per function of a batch its probability, its pooled embedding and its top-k statements, written to a device
// result store at a device cursor, so that captured replays append (include/ddfa_b200.h, K9'').
//
// Ranking: the rule of ddfa_stmt_metric (csrc/statements.cu) and of Python's stable sorted(..., reverse=True): score descending,
// equal scores in node order, with NaN after every number (-inf included) and NaNs in node order.  Each node gets a 64-bit key,
// larger = ranked ahead: the high word orders the score (-0.0 folded onto +0.0, which compares equal; NaN lowest), the low word is
// ~local_id (lower id ahead).  Keys are unique within a function, so rank j is the j-th largest key: round j takes the maximum key
// below the one of round j - 1, over every node of the function.  min(k, nodes) rounds, each one pass over the function's scores
// and a CTA reduction; exact, no atomics, and nothing depends on scheduling.
//
// Order: one CTA per function (grid-stride over a grid of min(num_graphs, kMaxCtas) CTAs).  Every CTA reads cursor[0] and writes
// positions cursor[0] + b; a second one-thread launch advances the cursor after them, in stream order.
#include <math.h>

#include "common.cuh"

namespace ddfa {
namespace predict {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCtas = 2 * kNumSMs;
constexpr int kMaxK = DDFA_PREDICT_MAX_K;

__device__ __forceinline__ unsigned long long rank_key(float s, int64_t local) {
  uint32_t hi = 0u;                                         // NaN: below every number
  if (!isnan(s)) {
    const uint32_t u = __float_as_uint(s == 0.f ? 0.f : s);  // -0.0 ties +0.0
    hi = (u & 0x80000000u) ? ~u : (u | 0x80000000u);         // -inf -> 0x007fffff > 0
  }
  return ((unsigned long long)hi << 32) | (unsigned long long)(0xffffffffu - (uint32_t)local);
}

__device__ __forceinline__ unsigned long long warp_max(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// functions stored by this call: b < stored lands at cursor[0] + b < capacity
__device__ __forceinline__ int32_t stored_count(int64_t base, int64_t capacity, int32_t num_valid) {
  const int64_t room = capacity - base;
  return room <= 0 ? 0 : (room < num_valid ? (int32_t)room : num_valid);
}

__global__ void __launch_bounds__(kThreads) store_kernel(const float *__restrict__ logits, const float *__restrict__ node_probs,
                                                         const float *__restrict__ pooled, int32_t out_dim,
                                                         const float *__restrict__ scores, int32_t k,
                                                         const int32_t *__restrict__ graph_ptr, int32_t num_valid,
                                                         float *__restrict__ prob_out, float *__restrict__ emb_out,
                                                         int32_t *__restrict__ top_idx, float *__restrict__ top_score,
                                                         const int64_t *__restrict__ cursor, int64_t capacity) {
  __shared__ unsigned long long s_key[2][kWarps];     // by round parity: one barrier per round
  __shared__ float s_max[kWarps];
  __shared__ int s_nan[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float qnan = __int_as_float(0x7fc00000);
  const int64_t base = cursor[0];
  const int32_t stored = stored_count(base, capacity, num_valid);
  for (int32_t b = blockIdx.x; b < stored; b += gridDim.x) {
    const int64_t p = base + b;
    const int64_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
    if (logits != nullptr && threadIdx.x == 0) prob_out[p] = 1.f / (1.f + expf(-logits[b]));    // eval_metrics.cu's p
    if (node_probs != nullptr) {
      // max over the function's nodes; a NaN anywhere makes the function's probability NaN; no node: 0
      float m = -INFINITY;
      int nan = 0;
      for (int64_t n = n0 + threadIdx.x; n < n1; n += kThreads) {
        const float v = node_probs[n];
        nan |= isnan(v) ? 1 : 0;
        m = fmaxf(m, v);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        nan |= __shfl_xor_sync(0xffffffffu, nan, o);
      }
      if (lane == 0) { s_max[warp] = m; s_nan[warp] = nan; }
      __syncthreads();
      if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 1; w < kWarps; ++w) { m = fmaxf(m, s_max[w]); nan |= s_nan[w]; }
        prob_out[p] = n1 == n0 ? 0.f : (nan ? qnan : m);
      }
    }
    if (emb_out != nullptr)
      for (int32_t c = threadIdx.x; c < out_dim; c += kThreads) emb_out[p * out_dim + c] = pooled[(int64_t)b * out_dim + c];
    if (k > 0) {
      const int64_t len = n1 - n0;
      const int32_t rounds = len < k ? (int32_t)len : k;
      unsigned long long bound = ~0ull;                 // above every key (the high word of a key is never 0xffffffff)
      for (int32_t j = 0; j < rounds; ++j) {
        unsigned long long best = 0ull;                 // below every key (the low word of a key is >= 2^31 - 1)
        for (int64_t n = n0 + threadIdx.x; n < n1; n += kThreads) {
          const unsigned long long key = rank_key(scores[n], n - n0);
          if (key < bound && key > best) best = key;
        }
        best = warp_max(best);
        if (lane == 0) s_key[j & 1][warp] = best;
        __syncthreads();
        best = s_key[j & 1][0];
#pragma unroll
        for (int w = 1; w < kWarps; ++w) best = s_key[j & 1][w] > best ? s_key[j & 1][w] : best;
        if (threadIdx.x == 0) {
          const int32_t local = (int32_t)(0xffffffffu - (uint32_t)best);
          top_idx[p * k + j] = local;
          top_score[p * k + j] = scores[n0 + local];    // the raw score (-0.0 and the NaN payload kept)
        }
        bound = best;
      }
      for (int32_t j = rounds + threadIdx.x; j < k; j += kThreads) {
        top_idx[p * k + j] = -1;
        top_score[p * k + j] = qnan;
      }
    }
    __syncthreads();      // the shared words are rewritten by the next function
  }
}

__global__ void advance_kernel(int64_t *__restrict__ cursor, int64_t capacity, int32_t num_valid) {
  const int64_t base = cursor[0];
  const int32_t stored = stored_count(base, capacity, num_valid);
  cursor[0] = base + stored;
  cursor[1] += num_valid - stored;
}

}  // namespace predict
}  // namespace ddfa

extern "C" {

int ddfa_predict_store(const float *logits, const float *node_probs, const float *pooled, int32_t out_dim, const float *scores, int32_t k,
                       const int32_t *graph_ptr, int32_t num_graphs, int32_t num_valid, float *prob_out, float *emb_out,
                       int32_t *top_idx_out, float *top_score_out, int64_t *cursor, int64_t capacity, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::predict;
  DDFA_REQUIRE(k >= 0 && k <= kMaxK, "ddfa_predict_store: k=%d not in [0, %d]", k, kMaxK);
  DDFA_REQUIRE(capacity >= 0, "ddfa_predict_store: capacity=%lld < 0", (long long)capacity);
  DDFA_REQUIRE(num_graphs >= 0 && num_valid >= 0 && num_valid <= num_graphs,
               "ddfa_predict_store: need 0 <= num_valid (%d) <= num_graphs (%d)", num_valid, num_graphs);
  DDFA_REQUIRE(!(logits && node_probs), "ddfa_predict_store: logits (graph style) and node_probs (node style) are alternatives");
  DDFA_REQUIRE((prob_out != nullptr) == (logits != nullptr || node_probs != nullptr),
               "ddfa_predict_store: prob_out is given exactly when logits or node_probs is");
  DDFA_REQUIRE((emb_out != nullptr) == (pooled != nullptr), "ddfa_predict_store: emb_out is given exactly when pooled is");
  DDFA_REQUIRE(pooled == nullptr || out_dim > 0, "ddfa_predict_store: out_dim=%d, need > 0 with pooled", out_dim);
  DDFA_REQUIRE((scores != nullptr) == (k > 0) && (top_idx_out != nullptr) == (k > 0) && (top_score_out != nullptr) == (k > 0),
               "ddfa_predict_store: scores, top_idx_out and top_score_out are given exactly when k > 0 (k=%d)", k);
  DDFA_REQUIRE(cursor != nullptr, "ddfa_predict_store: NULL cursor");
  DDFA_REQUIRE((reinterpret_cast<uintptr_t>(cursor) & 7u) == 0, "ddfa_predict_store: cursor must be 8-byte aligned");
  if (num_valid == 0) return DDFA_OK;
  DDFA_REQUIRE(graph_ptr != nullptr, "ddfa_predict_store: NULL graph_ptr");
  cudaStream_t stream = as_stream(stream_);
  const int ctas = num_graphs > kMaxCtas ? kMaxCtas : num_graphs;
  store_kernel<<<ctas, kThreads, 0, stream>>>(logits, node_probs, pooled, out_dim, scores, k, graph_ptr, num_valid, prob_out, emb_out,
                                              top_idx_out, top_score_out, cursor, capacity);
  DDFA_CHECK_LAUNCH("predict_store_kernel");
  advance_kernel<<<1, 1, 0, stream>>>(cursor, capacity, num_valid);
  DDFA_CHECK_LAUNCH("predict_advance_kernel");
  return DDFA_OK;
}

}  // extern "C"
