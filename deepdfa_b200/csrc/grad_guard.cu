// Gradient guard for the fused optimizer step: the total L2 norm of the flat gradient buffer, gradient-norm clipping and
// skipping of non-finite steps (torch.nn.utils.clip_grad_norm_ + GradScaler's skip rule, grad_guard.cuh), as two launches
// before a guarded form of K10's Adam.  Everything is read from device memory when it runs, so the whole sequence is
// CUDA-graph capturable and a captured step sees later writes of max_norm.
#include "common.cuh"
#include "grad_guard.cuh"

namespace ddfa {
namespace guard {

// A FIXED grid, whatever the buffer size or the device: the partials and their order depend on numel and the pointer's alignment
// only, so the norm is the same in both tuning modes and from call to call.
constexpr int kCtas = 128, kThreads = 256;

// per-CTA fp64 sum of squares: 16-byte unit u (then the scalar tail) goes to thread u % (kCtas * kThreads), which adds its units
// in increasing order; the CTA then adds its threads' sums in a fixed tree
__global__ void __launch_bounds__(kThreads) sumsq_partials_kernel(const float *__restrict__ g, int64_t n, int64_t n4,
                                                                  double *__restrict__ partials) {
  __shared__ double s[kThreads];
  const int64_t tid = (int64_t)blockIdx.x * kThreads + threadIdx.x, stride = (int64_t)kCtas * kThreads;
  double acc = 0.0;
  for (int64_t u = tid; u < n4; u += stride) {
    const float4 v = __ldcs(reinterpret_cast<const float4 *>(g) + u);
    acc += sq(v.x);
    acc += sq(v.y);
    acc += sq(v.z);
    acc += sq(v.w);
  }
  for (int64_t i = 4 * n4 + tid; i < n; i += stride) acc += sq(g[i]);
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partials[blockIdx.x] = s[0];
}

// the partials added in CTA order, then norm / coef / flag (one thread: 128 dependent adds)
__global__ void sumsq_finish_kernel(const double *__restrict__ partials, const float *__restrict__ max_norm, float *__restrict__ gstate) {
  double s = 0.0;
  for (int c = 0; c < kCtas; ++c) s += partials[c];
  float norm, coef;
  bool nonfinite;
  finish(s, max_norm, &norm, &coef, &nonfinite);
  gstate[kNorm] = norm;
  gstate[kCoef] = coef;
  gstate[kNonFinite] = nonfinite ? 1.f : 0.f;
}

// adam_flat_kernel (loss_adam.cu) with g * coef in place of g.  skipped != NULL and a non-finite norm: the CTA writes nothing.
// coef == 1 gives g * 1 == g, so the update is then bit-identical to adam_flat_kernel's.
__global__ void __launch_bounds__(256) adam_flat_guarded_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                                                                float *__restrict__ v, const int32_t *__restrict__ step_count, int64_t n,
                                                                const float *__restrict__ hyper, const float *__restrict__ gstate,
                                                                const int32_t *__restrict__ skipped) {
  if (skipped && gstate[kNonFinite] != 0.f) return;
  const float lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2], eps = hyper[3], wd = hyper[4];
  const float coef = gstate[kCoef];
  __shared__ float s_c[2];
  if (threadIdx.x == 0) {
    const double t = (double)(*step_count + 1);
    const double bc1 = 1.0 - pow((double)beta1, t);
    const double bc2 = 1.0 - pow((double)beta2, t);
    s_c[0] = (float)((double)lr / bc1);   // step_size
    s_c[1] = (float)sqrt(bc2);            // bias_correction2_sqrt
  }
  __syncthreads();
  const float step_size = s_c[0], bc2s = s_c[1];
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float gi = g[i] * coef;                              // clip_grad_norm_: grad.mul_(clip_coef_clamped)
  const float pi = p[i];
  gi = fmaf(wd, pi, gi);                               // grad = grad + wd * param  (coupled L2)
  const float mi = fmaf(beta1, m[i], (1.f - beta1) * gi);  // exp_avg.lerp_(grad, 1-beta1)
  const float vi = fmaf(beta2, v[i], (1.f - beta2) * gi * gi);
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) / bc2s + eps;
  p[i] = pi - step_size * (mi / denom);
}

// a skipped step leaves the Adam step counter alone (torch counts the optimizer.step() calls that happened) and counts the skip
__global__ void adam_step_inc_guarded_kernel(int32_t *step_count, const float *gstate, int32_t *skipped) {
  if (skipped && gstate[kNonFinite] != 0.f)
    *skipped += 1;
  else
    *step_count += 1;
}

}  // namespace guard
}  // namespace ddfa

extern "C" {

size_t ddfa_grad_norm_workspace_bytes(int64_t numel) {
  (void)numel;
  return sizeof(double) * ddfa::guard::kCtas;
}

int ddfa_grad_norm(const float *grads, int64_t numel, const float *max_norm, float *gstate, void *workspace, size_t workspace_bytes,
                   void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0, "ddfa_grad_norm: negative numel");
  DDFA_REQUIRE((grads || numel == 0) && gstate && workspace, "ddfa_grad_norm: NULL pointer");
  DDFA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "ddfa_grad_norm: workspace must be 8-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_grad_norm_workspace_bytes(numel), "ddfa_grad_norm: workspace of %zu bytes, need %zu", workspace_bytes,
               ddfa_grad_norm_workspace_bytes(numel));
  cudaStream_t stream = as_stream(stream_);
  double *partials = static_cast<double *>(workspace);
  const int64_t n4 = (grads && aligned16(grads)) ? numel >> 2 : 0;
  guard::sumsq_partials_kernel<<<guard::kCtas, guard::kThreads, 0, stream>>>(grads, numel, n4, partials);
  DDFA_CHECK_LAUNCH("sumsq_partials_kernel");
  guard::sumsq_finish_kernel<<<1, 1, 0, stream>>>(partials, max_norm, gstate);
  DDFA_CHECK_LAUNCH("sumsq_finish_kernel");
  return DDFA_OK;
}

int ddfa_adam_flat_guarded(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                           const float *hyper, const float *gstate, int32_t *skipped, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(numel >= 0, "ddfa_adam_flat_guarded: negative numel");
  DDFA_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_count && hyper && gstate, "ddfa_adam_flat_guarded: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  if (numel > 0) {
    guard::adam_flat_guarded_kernel<<<(unsigned)((numel + 255) / 256), 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, step_count,
                                                                                        numel, hyper, gstate, skipped);
    DDFA_CHECK_LAUNCH("adam_flat_guarded_kernel");
  }
  guard::adam_step_inc_guarded_kernel<<<1, 1, 0, stream>>>(step_count, gstate, skipped);
  DDFA_CHECK_LAUNCH("adam_step_inc_guarded_kernel");
  return DDFA_OK;
}

}  // extern "C"
