// Evaluation metrics accumulated on the device: one batch's logits -> confusion counts, the batch's mean BCE and (optionally) the
// stored probabilities / labels, added to a persistent fp64 metric state (layout in include/ddfa_b200.h).
//
// Reference: BaseModule.validation_step / test_step (base_module.py:211-224,238-323) feed sigmoid(out) and the labels into
// torchmetrics (Accuracy / Precision / Recall / F1Score, micro, threshold 0.5) and CatMetric (test_preds / test_labels); the
// epoch ends (base_module.py:325-346) compute them.  Here nothing syncs with the host: every grid is sized from the capacity (B
// graphs or N rows), the row count S and the store offset are read on the device, so one captured CUDA graph serves every batch
// of a bucket shape.
//
// Order: each CTA reduces its samples (integer counts as exact fp64 integers, the loss terms in fp64) with a fixed shuffle tree and
// writes one partial; a one-thread launch adds the partials in CTA order and updates the state.  The grid depends on the capacity
// only, so the state is bit-reproducible in both tuning modes.
#include <math.h>

#include "common.cuh"

namespace ddfa {
namespace evalm {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCtas = 2 * kNumSMs;
constexpr int kFields = 5;          // per-CTA partial: loss sum, TP, FP, TN, FN
enum { kTP = 0, kFP = 1, kTN = 2, kFN = 3, kSamples = 4, kBatches = 5, kLossW = 6, kWeight = 7, kStored = 8, kOverflow = 9 };

struct Acc {
  double loss = 0.0, tp = 0.0, fp = 0.0, tn = 0.0, fn = 0.0;
};

// one sample: the loss term of graph_label_bce_kernel, p as loss_adam.cu / torch.sigmoid compute it, prediction p >= 0.5
__device__ __forceinline__ void add_sample(Acc &a, float x, float y, float pos_weight, int64_t pos, float *probs_out, float *labels_out,
                                           int64_t capacity) {
  const float lw = 1.f + (pos_weight - 1.f) * y;
  const float term = (1.f - y) * x + lw * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f));
  const float p = 1.f / (1.f + expf(-x));
  const bool pred = p >= 0.5f, truth = y != 0.f;
  a.loss += (double)term;
  a.tp += (pred && truth) ? 1.0 : 0.0;
  a.fp += (pred && !truth) ? 1.0 : 0.0;
  a.tn += (!pred && !truth) ? 1.0 : 0.0;
  a.fn += (!pred && truth) ? 1.0 : 0.0;
  if (probs_out && pos < capacity) {
    probs_out[pos] = p;
    labels_out[pos] = y;
  }
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the CTA's five sums in a fixed order (shuffle tree per warp, warps in order) -> partials[blockIdx.x]
__device__ __forceinline__ void write_partial(Acc a, double *__restrict__ partials) {
  __shared__ double s[kWarps][kFields];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double v[kFields] = {warp_sum_f64(a.loss), warp_sum_f64(a.tp), warp_sum_f64(a.fp), warp_sum_f64(a.tn), warp_sum_f64(a.fn)};
  if (lane == 0) {
#pragma unroll
    for (int f = 0; f < kFields; ++f) s[warp][f] = v[f];
  }
  __syncthreads();
  if (threadIdx.x < kFields) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += s[w][threadIdx.x];
    partials[blockIdx.x * kFields + threadIdx.x] = t;
  }
}

// graph form: warp per graph (grid-stride over the valid graphs), label = max of vuln over the graph's nodes
__global__ void __launch_bounds__(kThreads) graph_metrics_kernel(const float *__restrict__ logits, const int32_t *__restrict__ vuln,
                                                                 const int32_t *__restrict__ graph_ptr, int32_t B_valid, float pos_weight,
                                                                 const double *__restrict__ state, float *__restrict__ probs_out,
                                                                 float *__restrict__ labels_out, int64_t capacity,
                                                                 double *__restrict__ partials) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)state[kStored];
  Acc a;
  for (int32_t b = blockIdx.x * kWarps + warp; b < B_valid; b += gridDim.x * kWarps) {
    const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
    int32_t mx = INT32_MIN;
    for (int32_t n = n0 + lane; n < n1; n += 32) mx = max(mx, vuln[n]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (n1 <= n0) mx = 0;
    if (lane == 0) add_sample(a, logits[b], (float)mx, pos_weight, base + b, probs_out, labels_out, capacity);
  }
  write_partial(a, partials);
}

// row form: thread per row s < S = *num_rows, label vuln[rows[s]]
__global__ void __launch_bounds__(kThreads) row_metrics_kernel(const float *__restrict__ logits, const int32_t *__restrict__ vuln,
                                                               const int32_t *__restrict__ rows, const int32_t *__restrict__ num_rows,
                                                               int32_t N, float pos_weight, const double *__restrict__ state,
                                                               float *__restrict__ probs_out, float *__restrict__ labels_out,
                                                               int64_t capacity, double *__restrict__ partials) {
  const int32_t S = min(max(*num_rows, 0), N);
  const int64_t base = (int64_t)state[kStored];
  Acc a;
  for (int32_t s = blockIdx.x * kThreads + threadIdx.x; s < S; s += gridDim.x * kThreads)
    add_sample(a, logits[s], (float)vuln[rows[s]], pos_weight, base + s, probs_out, labels_out, capacity);
  write_partial(a, partials);
}

// the partials in CTA order, then the state: counts, the batch's mean loss times its weight, the store offset and overflow
__global__ void metrics_finish_kernel(const double *__restrict__ partials, int ctas, double weight, int64_t capacity, int store,
                                      double *__restrict__ state) {
  double t[kFields] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int c = 0; c < ctas; ++c) {
#pragma unroll
    for (int f = 0; f < kFields; ++f) t[f] += partials[c * kFields + f];
  }
  const double n = t[1] + t[2] + t[3] + t[4];
  state[kTP] += t[1];
  state[kFP] += t[2];
  state[kTN] += t[3];
  state[kFN] += t[4];
  state[kSamples] += n;
  state[kBatches] += 1.0;
  if (n > 0.0) {
    state[kLossW] += (t[0] / n) * weight;
    state[kWeight] += weight;
  }
  if (store) {
    const double stored = state[kStored];
    const double kept = fmin((double)capacity, stored + n);
    state[kStored] = fmax(kept, stored);
    state[kOverflow] += stored + n - fmax(kept, stored);
  }
}

inline int ctas_for(int64_t units, int per_cta) {
  const int64_t c = (units + per_cta - 1) / per_cta;
  return (int)(c < 1 ? 1 : (c > kMaxCtas ? kMaxCtas : c));
}

int finish(const double *partials, int ctas, double weight, int64_t capacity, bool store, double *state, cudaStream_t stream) {
  metrics_finish_kernel<<<1, 1, 0, stream>>>(partials, ctas, weight, capacity, store ? 1 : 0, state);
  DDFA_CHECK_LAUNCH("metrics_finish_kernel");
  return DDFA_OK;
}

}  // namespace evalm
}  // namespace ddfa

extern "C" {

size_t ddfa_eval_metrics_workspace_bytes(void) { return sizeof(double) * ddfa::evalm::kFields * ddfa::evalm::kMaxCtas; }

#define DDFA_EVAL_COMMON_CHECKS(fn)                                                                                                   \
  DDFA_REQUIRE(state && workspace, fn ": NULL pointer");                                                                              \
  DDFA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0 && (reinterpret_cast<uintptr_t>(state) & 7u) == 0,                 \
               fn ": state and workspace must be 8-byte aligned");                                                                    \
  DDFA_REQUIRE(workspace_bytes >= ddfa_eval_metrics_workspace_bytes(), fn ": workspace of %zu bytes, need %zu", workspace_bytes,      \
               ddfa_eval_metrics_workspace_bytes());                                                                                  \
  DDFA_REQUIRE(capacity >= 0 && ((probs_out == nullptr) == (labels_out == nullptr)),                                                  \
               fn ": capacity (%lld) < 0, or only one of probs_out / labels_out given", (long long)capacity);                        \
  DDFA_REQUIRE(isfinite(weight) && weight >= 0.0, fn ": weight must be finite and >= 0")

int ddfa_eval_metrics_graph(const float *logits, const int32_t *vuln, const int32_t *graph_ptr, int32_t num_graphs, int32_t num_valid,
                            float pos_weight, double weight, double *state, float *probs_out, float *labels_out, int64_t capacity,
                            void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::evalm;
  DDFA_REQUIRE(num_graphs >= 0 && num_valid >= 0 && num_valid <= num_graphs,
               "ddfa_eval_metrics_graph: need 0 <= num_valid (%d) <= num_graphs (%d)", num_valid, num_graphs);
  DDFA_EVAL_COMMON_CHECKS("ddfa_eval_metrics_graph");
  DDFA_REQUIRE(num_valid == 0 || (logits && vuln && graph_ptr), "ddfa_eval_metrics_graph: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  double *partials = static_cast<double *>(workspace);
  const int ctas = ctas_for(num_graphs, kWarps);
  graph_metrics_kernel<<<ctas, kThreads, 0, stream>>>(logits, vuln, graph_ptr, num_valid, pos_weight, state, probs_out, labels_out, capacity,
                                                      partials);
  DDFA_CHECK_LAUNCH("graph_metrics_kernel");
  return finish(partials, ctas, weight, capacity, probs_out != nullptr, state, stream);
}

int ddfa_eval_metrics_rows(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows, int32_t num_nodes,
                           float pos_weight, double weight, double *state, float *probs_out, float *labels_out, int64_t capacity,
                           void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::evalm;
  DDFA_REQUIRE(num_nodes >= 0, "ddfa_eval_metrics_rows: num_nodes=%d < 0", num_nodes);
  DDFA_EVAL_COMMON_CHECKS("ddfa_eval_metrics_rows");
  DDFA_REQUIRE(num_rows && (num_nodes == 0 || (logits && vuln && rows)), "ddfa_eval_metrics_rows: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  double *partials = static_cast<double *>(workspace);
  const int ctas = ctas_for(num_nodes, kThreads);
  row_metrics_kernel<<<ctas, kThreads, 0, stream>>>(logits, vuln, rows, num_rows, num_nodes, pos_weight, state, probs_out, labels_out,
                                                    capacity, partials);
  DDFA_CHECK_LAUNCH("row_metrics_kernel");
  return finish(partials, ctas, weight, capacity, probs_out != nullptr, state, stream);
}

}  // extern "C"
