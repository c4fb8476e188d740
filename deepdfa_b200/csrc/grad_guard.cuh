// Gradient guard arithmetic shared by ddfa_grad_norm (grad_guard.cu) and the guarded peer-memory exchange (allreduce_adam.cu).
//
// The guard is torch.nn.utils.clip_grad_norm_(params, max_norm, norm_type=2) followed by GradScaler's rule for a non-finite step
// (optimizer.step() is not called):
//   norm = sqrt(sum g^2)                      squares summed in fp64 in a fixed order, rounded ONCE to fp32
//   coef = min(1, max_norm / (norm + 1e-6))   in fp32 from the fp32 norm, as torch computes it (NaN stays NaN)
//   skip = !isfinite(norm)                    honoured only when the caller asks for skipping
// fp32 squares are exact in fp64, and 2^24 squares of FLT_MAX still sum to a finite fp64 value, so the norm is finite whenever
// every gradient is finite and the norm itself is at most FLT_MAX (torch's fp32 sum overflows to inf from ~1e19 per element).
#pragma once

#include <math.h>

namespace ddfa {
namespace guard {

// gstate words: [0] fp32 norm, [1] fp32 coef, [2] 1.0f when the norm is not finite, else 0.0f
constexpr int kNorm = 0, kCoef = 1, kNonFinite = 2;

__device__ __forceinline__ double sq(float x) { return (double)x * (double)x; }

// max_norm: NULL or one device float read now (so a captured launch sees later writes); NULL / +inf = measure, don't clip
__device__ __forceinline__ void finish(double sumsq, const float *max_norm, float *norm_out, float *coef_out, bool *nonfinite_out) {
  const float norm = (float)sqrt(sumsq);
  const float mx = max_norm ? *max_norm : INFINITY;
  const float c = __fdiv_rn(mx, __fadd_rn(norm, 1e-6f));
  *norm_out = norm;
  *coef_out = c > 1.f ? 1.f : c;            // torch.clamp(max=1): a NaN coefficient stays NaN
  *nonfinite_out = !isfinite(norm);
}

}  // namespace guard
}  // namespace ddfa
