// Gradient guard for the fused optimizer step: the total L2 norm of the flat gradient buffer and the clipping coefficient and
// skip flag derived from it (torch.nn.utils.clip_grad_norm_ + GradScaler's skip rule, adam.cuh), as two launches before the
// guarded form of K10's Adam (ddfa_adam_flat_guarded, loss_adam.cu), which reads them.  Everything is read from device memory
// when it runs, so the whole sequence is CUDA-graph capturable and a captured step sees later writes of max_norm.
#include "common.cuh"
#include "adam.cuh"

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

}  // extern "C"
