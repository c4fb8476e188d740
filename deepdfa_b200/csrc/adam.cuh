// The optimizer arithmetic, written once for every Adam entry point: the flat update (loss_adam.cu), the peer-memory exchange
// (allreduce_adam.cu) and the gradient guard (grad_guard.cu).
//
// Adam is torch.optim.Adam with coupled L2 (DDFA/configs/config_default.yaml:43-47); the grouped entry points also run the
// decoupled form of torch.optim.AdamW per parameter group (update_decoupled, below).  Every entry point computes
// bit-identical results from the same inputs, so the expression order below must not change: a reordered or re-rounded term
// changes parameters in the last bits.
//
// The guard is torch.nn.utils.clip_grad_norm_(params, max_norm, norm_type=2) followed by GradScaler's rule for a non-finite step
// (optimizer.step() is not called):
//   norm = sqrt(sum g^2)                      squares summed in fp64 in a fixed order, rounded ONCE to fp32
//   coef = min(1, max_norm / (norm + 1e-6))   in fp32 from the fp32 norm, as torch computes it (NaN stays NaN)
//   skip = !isfinite(norm)                    honoured only when the caller asks for skipping
// fp32 squares are exact in fp64, and 2^24 squares of FLT_MAX still sum to a finite fp64 value, so the norm is finite whenever
// every gradient is finite and the norm itself is at most FLT_MAX (torch's fp32 sum overflows to inf from ~1e19 per element).
// Adam then runs on g * coef; the unguarded kernels never multiply by a coefficient.
#pragma once

#include <math.h>
#include <stdint.h>

namespace ddfa {
namespace adam {

struct Hyper {
  float lr, beta1, beta2, eps, wd;
};

// hyper: NULL (the by-value h is used) or 5 device floats [lr, beta1, beta2, eps, wd] read when the kernel runs, so a captured
// launch sees values written after the capture
__device__ __forceinline__ Hyper load(Hyper h, const float *hyper) {
  if (hyper) h = Hyper{hyper[0], hyper[1], hyper[2], hyper[3], hyper[4]};
  return h;
}

// torch's bias correction for step t = step + 1, in fp64: step_size = lr / (1 - beta1^t), bc2s = sqrt(1 - beta2^t)
struct Bias {
  float step_size, bc2s;
};
__device__ __forceinline__ Bias bias_correction(float lr, float beta1, float beta2, int32_t step) {
  const double t = (double)(step + 1);
  const double bc1 = 1.0 - pow((double)beta1, t);
  const double bc2 = 1.0 - pow((double)beta2, t);
  return Bias{(float)((double)lr / bc1), (float)sqrt(bc2)};
}

// one element: gradient g -> parameter p, moments m and v
__device__ __forceinline__ void update(float g, float &p, float &m, float &v, const Hyper &h, const Bias &c) {
  const float gi = fmaf(h.wd, p, g);                  // grad = grad + wd * param  (coupled L2)
  m = fmaf(h.beta1, m, (1.f - h.beta1) * gi);         // exp_avg.lerp_(grad, 1-beta1)
  v = fmaf(h.beta2, v, (1.f - h.beta2) * gi * gi);
  const float denom = sqrtf(v) / c.bc2s + h.eps;
  p = p - c.step_size * (m / denom);
}
__device__ __forceinline__ void update(const float4 &g, float4 &p, float4 &m, float4 &v, const Hyper &h, const Bias &c) {
  update(g.x, p.x, m.x, v.x, h, c);
  update(g.y, p.y, m.y, v.y, h, c);
  update(g.z, p.z, m.z, v.z, h, c);
  update(g.w, p.w, m.w, v.w, h, c);
}

// Decoupled weight decay: torch.optim.AdamW / Adam(decoupled_weight_decay=True), torch/optim/adam.py _single_tensor_adam:
//   param.mul_(1 - lr * weight_decay)            decay = fp32(1 - lr * wd), computed by the host in fp64 and rounded once
// then the moments and the step exactly as in update() with no wd * p term in the gradient.  decay == 1 (wd == 0) leaves p as is.
__device__ __forceinline__ void update_decoupled(float g, float &p, float &m, float &v, const Hyper &h, float decay, const Bias &c) {
  p = p * decay;
  m = fmaf(h.beta1, m, (1.f - h.beta1) * g);
  v = fmaf(h.beta2, v, (1.f - h.beta2) * g * g);
  const float denom = sqrtf(v) / c.bc2s + h.eps;
  p = p - c.step_size * (m / denom);
}

// ---- parameter groups: a device table of G rows of kGroupWords floats, read when the kernel runs
constexpr int kMaxGroups = 64;
constexpr int kGroupWords = 8;
enum GroupWord { kLr = 0, kBeta1, kBeta2, kEps, kWd, kDecoupled, kDecay, kPad };

struct Group {
  Hyper h;
  float decay;       // decoupled groups: fp32(1 - lr * wd); coupled groups: unused
  bool decoupled;
};
__device__ __forceinline__ Group load_group(const float *row) {
  return Group{Hyper{row[kLr], row[kBeta1], row[kBeta2], row[kEps], row[kWd]}, row[kDecay], row[kDecoupled] != 0.f};
}
// one element of a group: the coupled form is update() itself, so a coupled group is bit-identical to the single-group kernels
__device__ __forceinline__ void update(float g, float &p, float &m, float &v, const Group &gr, const Bias &c) {
  if (gr.decoupled)
    update_decoupled(g, p, m, v, gr.h, gr.decay, c);
  else
    update(g, p, m, v, gr.h, c);
}
__device__ __forceinline__ void update(const float4 &g, float4 &p, float4 &m, float4 &v, const Group &gr, const Bias &c) {
  update(g.x, p.x, m.x, v.x, gr, c);
  update(g.y, p.y, m.y, v.y, gr, c);
  update(g.z, p.z, m.z, v.z, gr, c);
  update(g.w, p.w, m.w, v.w, gr, c);
}

// Threads [0, num_groups) of the CTA load the table into shared memory and compute each group's bias correction (fp64, from the
// one shared step count); the caller synchronises before reading.
__device__ __forceinline__ void load_groups(const float *__restrict__ table, int32_t num_groups, int32_t step, Group *s_g, Bias *s_c) {
  if ((int)threadIdx.x < num_groups) {
    const Group gr = load_group(table + (size_t)threadIdx.x * kGroupWords);
    s_g[threadIdx.x] = gr;
    s_c[threadIdx.x] = bias_correction(gr.h.lr, gr.h.beta1, gr.h.beta2, step);
  }
}

}  // namespace adam

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
