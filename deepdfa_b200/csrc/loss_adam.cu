// K8 — graph labels + BCE-with-logits loss (+ d loss / d logits), and K10 — fused Adam.
//
// K8 replaces BaseModule.get_label (base_module.py:83-95: dgl.unbatch + a Python loop taking
// max(_VULN) per graph) and torch.nn.BCEWithLogitsLoss(pos_weight) (base_module.py:72-74,183).
// K10 replaces torch.optim.Adam(lr=1e-3, weight_decay=1e-2) — coupled L2, not AdamW
// (DDFA/configs/config_default.yaml:43-47) — over one flat parameter buffer, with the hyperparameters by value
// (ddfa_adam_flat) or from a device word (ddfa_adam_flat_hp); ddfa_adam_flat_guarded is the same update on the clipped
// gradient, after ddfa_grad_norm (grad_guard.cu); ddfa_adam_flat_ranges updates only the elements inside a list of ranges (the
// trainable parameters of a partly frozen model); ddfa_adam_flat_groups gives every range a parameter group of its own
// hyperparameters, coupled (Adam) or decoupled (AdamW) weight decay.  The arithmetic is adam.cuh's.
#include <math.h>

#include "common.cuh"
#include "adam.cuh"

namespace ddfa {

// warp per graph: segment max of vuln, then the loss term of that graph
__global__ void __launch_bounds__(256) graph_label_bce_kernel(const float *__restrict__ logits, const int32_t *__restrict__ vuln,
                                                              const int32_t *__restrict__ graph_ptr, int32_t B, int32_t B_valid,
                                                              float pos_weight, float loss_scale, float grad_scale, float *__restrict__ labels,
                                                              float *__restrict__ loss_out, float *__restrict__ dlogits) {
  __shared__ float s_loss[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * 8 + warp;
  float term = 0.f;
  if (b < B) {
    const int32_t n0 = graph_ptr[b], n1 = graph_ptr[b + 1];
    int32_t mx = INT32_MIN;
    for (int32_t n = n0 + lane; n < n1; n += 32) mx = max(mx, vuln[n]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (n1 <= n0) mx = 0;  // empty graph: no label information
    const float y = (float)mx;
    if (lane == 0) {
      if (labels) labels[b] = y;
      if (dlogits && b >= B_valid) dlogits[b] = 0.f;      // padding graphs (shape bucketing): no loss term, no gradient
      if (logits && b < B_valid) {
        const float x = logits[b];
        // torch: (1-y)*x + (1+(pw-1)*y) * (log1p(exp(-|x|)) + max(-x,0))
        const float lw = 1.f + (pos_weight - 1.f) * y;
        term = (1.f - y) * x + lw * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f));
        if (dlogits) {
          const float sg = 1.f / (1.f + expf(-x));
          // d/dx = (1-y) - lw * (1 - sigmoid(x)) = sigmoid(x)*lw - y*pw ... expanded for clarity:
          dlogits[b] = grad_scale * ((1.f - y) - lw * (1.f - sg));
        }
      }
    }
  }
  if (lane == 0) s_loss[warp] = term;
  __syncthreads();
  if (threadIdx.x == 0 && loss_out) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_loss[w];
    atomicAdd(loss_out, loss_scale * s);
  }
}

// deterministic mode: the loss as one CTA's sum of the graphs' terms in a fixed order, from the labels graph_label_bce_kernel wrote
__global__ void __launch_bounds__(256) bce_loss_sum_kernel(const float *__restrict__ logits, const float *__restrict__ labels, int32_t B_valid,
                                                           float pos_weight, float loss_scale, float *__restrict__ loss_out) {
  __shared__ float s_t[256];
  float acc = 0.f;
  for (int32_t b = threadIdx.x; b < B_valid; b += 256) {
    const float x = logits[b], y = labels[b];
    const float lw = 1.f + (pos_weight - 1.f) * y;
    acc += (1.f - y) * x + lw * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f));
  }
  s_t[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_t[threadIdx.x] += s_t[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss_out = loss_scale * s_t[0];
}

// i inside one of the sorted, disjoint [begin, end) pairs of ranges[2 * num_ranges] (binary search for the last begin <= i)
__device__ __forceinline__ bool in_ranges(const int64_t *__restrict__ ranges, int32_t num_ranges, int64_t i) {
  int32_t lo = 0, hi = num_ranges;
  while (lo < hi) {
    const int32_t mid = (lo + hi) >> 1;
    if (ranges[2 * mid] <= i) lo = mid + 1;
    else hi = mid;
  }
  return lo > 0 && i < ranges[2 * lo - 1];
}

// Guarded: Adam on g * gstate[kCoef] (grad_guard.cu computed it); with skipped != NULL and a non-finite norm the CTA writes nothing.
// ranges != NULL: elements outside the ranges are neither read nor written.
template <bool Guarded>
__global__ void __launch_bounds__(256) adam_flat_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                                                        float *__restrict__ v, const int32_t *__restrict__ step_count, int64_t n,
                                                        adam::Hyper h, const float *__restrict__ hyper, const float *__restrict__ gstate,
                                                        const int32_t *__restrict__ skipped, const int64_t *__restrict__ ranges,
                                                        int32_t num_ranges) {
  if constexpr (Guarded) {
    if (skipped && gstate[guard::kNonFinite] != 0.f) return;
  }
  h = adam::load(h, hyper);
  __shared__ adam::Bias s_c;
  if (threadIdx.x == 0) s_c = adam::bias_correction(h.lr, h.beta1, h.beta2, *step_count);
  __syncthreads();
  const adam::Bias c = s_c;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n || (ranges && !in_ranges(ranges, num_ranges, i))) return;
  float gi = g[i];
  if constexpr (Guarded) gi = gi * gstate[guard::kCoef];     // clip_grad_norm_: grad.mul_(clip_coef_clamped)
  float pi = p[i], mi = m[i], vi = v[i];
  adam::update(gi, pi, mi, vi, h, c);
  m[i] = mi;
  v[i] = vi;
  p[i] = pi;
}

static_assert(adam::kMaxGroups == DDFA_ADAM_MAX_GROUPS && adam::kGroupWords == DDFA_ADAM_GROUP_WORDS, "group table layout");

// The range of ranges[3 * num_ranges] (sorted, disjoint [begin, end, group] triples) holding i, or -1 (binary search as in_ranges)
__device__ __forceinline__ int32_t find_range(const int64_t *__restrict__ ranges, int32_t num_ranges, int64_t i) {
  int32_t lo = 0, hi = num_ranges;
  while (lo < hi) {
    const int32_t mid = (lo + hi) >> 1;
    if (ranges[3 * mid] <= i) lo = mid + 1;
    else hi = mid;
  }
  return (lo > 0 && i < ranges[3 * lo - 2]) ? lo - 1 : -1;
}

// Parameter groups: element i inside range r is updated with the hyperparameters of group ranges[3r + 2] (a row of the table,
// adam::kGroupWords floats) and that group's bias correction; elements outside every range, or of a range whose group index is
// not in [0, num_groups), are neither read nor written.  Guarded as adam_flat_kernel.
template <bool Guarded>
__global__ void __launch_bounds__(256) adam_flat_groups_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                                                               float *__restrict__ v, const int32_t *__restrict__ step_count, int64_t n,
                                                               const int64_t *__restrict__ ranges, int32_t num_ranges,
                                                               const float *__restrict__ table, int32_t num_groups,
                                                               const float *__restrict__ gstate, const int32_t *__restrict__ skipped) {
  if constexpr (Guarded) {
    if (skipped && gstate[guard::kNonFinite] != 0.f) return;
  }
  __shared__ adam::Group s_g[adam::kMaxGroups];
  __shared__ adam::Bias s_c[adam::kMaxGroups];
  adam::load_groups(table, num_groups, *step_count, s_g, s_c);
  __syncthreads();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t r = find_range(ranges, num_ranges, i);
  if (r < 0) return;
  const int64_t grp = ranges[3 * r + 2];
  if (grp < 0 || grp >= num_groups) return;
  float gi = g[i];
  if constexpr (Guarded) gi = gi * gstate[guard::kCoef];     // clip_grad_norm_: grad.mul_(clip_coef_clamped)
  float pi = p[i], mi = m[i], vi = v[i];
  adam::update(gi, pi, mi, vi, s_g[grp], s_c[grp]);
  m[i] = mi;
  v[i] = vi;
  p[i] = pi;
}

// gstate == NULL: the step.  Otherwise, with skipped != NULL and a non-finite norm, the skip counter instead: a skipped step
// leaves the Adam step count alone (torch counts the optimizer.step() calls that happened).
__global__ void adam_step_inc_kernel(int32_t *step_count, const float *gstate, int32_t *skipped) {
  if (gstate && skipped && gstate[guard::kNonFinite] != 0.f)
    *skipped += 1;
  else
    *step_count += 1;
}

int adam_step_inc_launch(int32_t *step_count, const float *gstate, int32_t *skipped, cudaStream_t stream) {
  adam_step_inc_kernel<<<1, 1, 0, stream>>>(step_count, gstate, skipped);
  DDFA_CHECK_LAUNCH("adam_step_inc_kernel");
  return DDFA_OK;
}

// the flat update and its step-count increment: two launches (none for the update when numel == 0)
template <bool Guarded>
static int adam_flat_launch(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                            adam::Hyper h, const float *hyper, const float *gstate, int32_t *skipped, void *stream_,
                            const int64_t *ranges = nullptr, int32_t num_ranges = 0) {
  cudaStream_t stream = as_stream(stream_);
  if (numel > 0) {
    adam_flat_kernel<Guarded><<<(unsigned)((numel + 255) / 256), 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, step_count, numel,
                                                                                  h, hyper, gstate, skipped, ranges, num_ranges);
    DDFA_CHECK_LAUNCH("adam_flat_kernel");
  }
  return adam_step_inc_launch(step_count, gstate, skipped, stream);
}

}  // namespace ddfa

extern "C" {

int ddfa_graph_label_bce_valid(const float *logits, const int32_t *vuln, const int32_t *graph_ptr, int32_t B, int32_t B_valid,
                               float pos_weight, float loss_scale, float grad_scale, float *labels, float *loss_out, float *dlogits,
                               void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(B >= 0 && B_valid >= 0 && B_valid <= B, "ddfa_graph_label_bce: need 0 <= num_valid (%d) <= num_graphs (%d)", B_valid, B);
  if (B == 0) return DDFA_OK;
  DDFA_REQUIRE(vuln && graph_ptr, "ddfa_graph_label_bce: NULL pointer");
  DDFA_REQUIRE(logits || (!loss_out && !dlogits), "ddfa_graph_label_bce: loss requested without logits");
  const bool det = deterministic() && loss_out != nullptr;      // the loss summed in a second, single-CTA pass over the labels
  DDFA_REQUIRE(!det || labels, "ddfa_graph_label_bce: in deterministic mode (DDFA_TUNE_DETERMINISTIC = 1) the loss needs the labels output");
  cudaStream_t stream = as_stream(stream_);
  if (loss_out) DDFA_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), stream));
  graph_label_bce_kernel<<<(B + 7) / 8, 256, 0, stream>>>(logits, vuln, graph_ptr, B, B_valid, pos_weight, loss_scale, grad_scale, labels,
                                                         det ? nullptr : loss_out, dlogits);
  DDFA_CHECK_LAUNCH("graph_label_bce_kernel");
  if (det) {
    bce_loss_sum_kernel<<<1, 256, 0, stream>>>(logits, labels, B_valid, pos_weight, loss_scale, loss_out);
    DDFA_CHECK_LAUNCH("bce_loss_sum_kernel");
  }
  return DDFA_OK;
}

int ddfa_graph_label_bce(const float *logits, const int32_t *vuln, const int32_t *graph_ptr, int32_t B, float pos_weight,
                         float loss_scale, float grad_scale, float *labels, float *loss_out, float *dlogits, void *stream_) {
  return ddfa_graph_label_bce_valid(logits, vuln, graph_ptr, B, B, pos_weight, loss_scale, grad_scale, labels, loss_out, dlogits, stream_);
}

int ddfa_adam_flat(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                   float lr, float beta1, float beta2, float eps, float weight_decay, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0, "ddfa_adam_flat: negative numel");
  DDFA_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_count, "ddfa_adam_flat: NULL pointer");
  return adam_flat_launch<false>(params, grads, exp_avg, exp_avg_sq, step_count, numel, adam::Hyper{lr, beta1, beta2, eps, weight_decay},
                                 nullptr, nullptr, nullptr, stream_);
}

int ddfa_adam_flat_hp(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                      const float *hyper, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0, "ddfa_adam_flat_hp: negative numel");
  DDFA_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_count && hyper, "ddfa_adam_flat_hp: NULL pointer");
  return adam_flat_launch<false>(params, grads, exp_avg, exp_avg_sq, step_count, numel, adam::Hyper{}, hyper, nullptr, nullptr, stream_);
}

int ddfa_adam_flat_guarded(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                           const float *hyper, const float *gstate, int32_t *skipped, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0, "ddfa_adam_flat_guarded: negative numel");
  DDFA_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_count && hyper && gstate, "ddfa_adam_flat_guarded: NULL pointer");
  return adam_flat_launch<true>(params, grads, exp_avg, exp_avg_sq, step_count, numel, adam::Hyper{}, hyper, gstate, skipped, stream_);
}

int ddfa_adam_flat_ranges(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                          const int64_t *ranges, int32_t num_ranges, const float *hyper, const float *gstate, int32_t *skipped, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0 && num_ranges >= 0, "ddfa_adam_flat_ranges: negative numel (%lld) or num_ranges (%d)", (long long)numel, num_ranges);
  DDFA_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_count && hyper && (ranges || num_ranges == 0),
               "ddfa_adam_flat_ranges: NULL pointer");
  DDFA_REQUIRE(gstate || !skipped, "ddfa_adam_flat_ranges: skipped given without gstate");
  if (num_ranges == 0) return adam_step_inc_launch(step_count, gstate, skipped, as_stream(stream_));   // nothing to update
  if (gstate)
    return adam_flat_launch<true>(params, grads, exp_avg, exp_avg_sq, step_count, numel, adam::Hyper{}, hyper, gstate, skipped, stream_,
                                  ranges, num_ranges);
  return adam_flat_launch<false>(params, grads, exp_avg, exp_avg_sq, step_count, numel, adam::Hyper{}, hyper, nullptr, nullptr, stream_,
                                 ranges, num_ranges);
}

int ddfa_adam_flat_groups(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                          const int64_t *ranges, int32_t num_ranges, const float *groups, int32_t num_groups, const float *gstate,
                          int32_t *skipped, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0 && num_ranges >= 0, "ddfa_adam_flat_groups: negative numel (%lld) or num_ranges (%d)", (long long)numel, num_ranges);
  DDFA_REQUIRE(num_groups >= 1 && num_groups <= adam::kMaxGroups, "ddfa_adam_flat_groups: num_groups (%d) must be in [1, %d]", num_groups,
               adam::kMaxGroups);
  DDFA_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_count && groups && (ranges || num_ranges == 0),
               "ddfa_adam_flat_groups: NULL pointer");
  DDFA_REQUIRE(gstate || !skipped, "ddfa_adam_flat_groups: skipped given without gstate");
  cudaStream_t stream = as_stream(stream_);
  if (numel > 0 && num_ranges > 0) {
    const unsigned blocks = (unsigned)((numel + 255) / 256);
    if (gstate)
      adam_flat_groups_kernel<true><<<blocks, 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, step_count, numel, ranges, num_ranges,
                                                                groups, num_groups, gstate, skipped);
    else
      adam_flat_groups_kernel<false><<<blocks, 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, step_count, numel, ranges, num_ranges,
                                                                 groups, num_groups, nullptr, nullptr);
    DDFA_CHECK_LAUNCH("adam_flat_groups_kernel");
  }
  return adam_step_inc_launch(step_count, gstate, skipped, stream);
}

}  // extern "C"
