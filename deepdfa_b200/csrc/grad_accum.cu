// Gradient accumulation over micro-batches (FusedTrainer(accumulate_grad_batches=k)): the flat fp32 gradient buffer of every
// micro-batch of a window is summed into an accumulator, and the window's last micro-batch adds the sum back into its own
// gradient buffer, so the exchange and the optimizer update read the window's sum where they always read the step's gradient.
// Elementwise, one 16-byte unit per thread and iteration: bit-reproducible by construction, in both tuning modes.
#include "common.cuh"

namespace ddfa {
namespace accum {

constexpr int kThreads = 256, kMaxCtas = 132 * 8;

template <int Mode>
__global__ void __launch_bounds__(kThreads) grad_accumulate_kernel(float4 *__restrict__ acc, float4 *__restrict__ g, int64_t n4) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t u = (int64_t)blockIdx.x * kThreads + threadIdx.x; u < n4; u += stride) {
    if (Mode == DDFA_GRAD_ACC_SET) {
      acc[u] = __ldcs(g + u);
    } else if (Mode == DDFA_GRAD_ACC_ADD) {
      const float4 a = acc[u], b = __ldcs(g + u);
      acc[u] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    } else {
      const float4 a = acc[u], b = g[u];
      g[u] = make_float4(b.x + a.x, b.y + a.y, b.z + a.z, b.w + a.w);
    }
  }
}

}  // namespace accum
}  // namespace ddfa

extern "C" {

int ddfa_grad_accumulate(float *acc, float *grads, int64_t begin, int64_t end, int32_t mode, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(mode == DDFA_GRAD_ACC_SET || mode == DDFA_GRAD_ACC_ADD || mode == DDFA_GRAD_ACC_APPLY,
               "ddfa_grad_accumulate: mode=%d is not DDFA_GRAD_ACC_SET / _ADD / _APPLY", mode);
  DDFA_REQUIRE(0 <= begin && begin <= end && begin % 4 == 0 && end % 4 == 0,
               "ddfa_grad_accumulate: range [%lld, %lld) must satisfy 0 <= begin <= end with both bounds multiples of 4",
               (long long)begin, (long long)end);
  if (begin == end) return DDFA_OK;
  DDFA_REQUIRE(acc && grads, "ddfa_grad_accumulate: NULL pointer");
  DDFA_REQUIRE(aligned16(acc) && aligned16(grads), "ddfa_grad_accumulate: acc and grads need 16-byte alignment");
  const int64_t n4 = (end - begin) / 4;
  const unsigned ctas = (unsigned)(n4 < (int64_t)accum::kMaxCtas * accum::kThreads ? (n4 + accum::kThreads - 1) / accum::kThreads
                                                                                     : accum::kMaxCtas);
  float4 *a = reinterpret_cast<float4 *>(acc + begin), *g = reinterpret_cast<float4 *>(grads + begin);
  cudaStream_t stream = as_stream(stream_);
  if (mode == DDFA_GRAD_ACC_SET)
    accum::grad_accumulate_kernel<DDFA_GRAD_ACC_SET><<<ctas, accum::kThreads, 0, stream>>>(a, g, n4);
  else if (mode == DDFA_GRAD_ACC_ADD)
    accum::grad_accumulate_kernel<DDFA_GRAD_ACC_ADD><<<ctas, accum::kThreads, 0, stream>>>(a, g, n4);
  else
    accum::grad_accumulate_kernel<DDFA_GRAD_ACC_APPLY><<<ctas, accum::kThreads, 0, stream>>>(a, g, n4);
  DDFA_CHECK_LAUNCH("grad_accumulate_kernel");
  return DDFA_OK;
}

}  // extern "C"
