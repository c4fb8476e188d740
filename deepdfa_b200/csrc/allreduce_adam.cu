// K10' — the data-parallel exchange FUSED with the optimizer, over NVLink peer memory (no NCCL call in the step).
//
// Replaces, for R ranks on one NVSwitch domain, the sequence "all-reduce of the flat gradient buffer; Adam on every rank"
// (reference: single-GPU `torch.optim.Adam`, DDFA/configs/config_default.yaml:43-47 — DDP is this repo's extension, SURVEY.md §8e)
// by ONE kernel per rank working on symmetric buffers every rank can address:
//
//   phase 1  "gradients complete": rank r tells every peer (a flag word in the PEER's memory, st.release.sys), then waits for
//            the R flags in its own memory (ld.acquire.sys).  The kernels that produced the gradients precede this launch in
//            stream order, so their writes are performed before the flag is.
//   reduce-scatter + Adam + all-gather in one pass: rank r owns the r-th 1/R of the flat buffers.  For its elements it sums the R
//            gradient copies straight out of the peers' memory (16-byte loads over NVLink, L1-bypassing), applies Adam with coupled L2
//            (moments live only on the owner: optimizer state is sharded), and stores the new parameters into EVERY rank's
//            parameter buffer (16-byte peer stores).  Bytes over the links per rank: (R-1)/R of the buffer in, the same out —
//            1.3 MB each way at R = 8 for the 1.5 MB buffer, against the 2 x 2(R-1)/R of a ring all-reduce plus its latency steps.
//   phase 2  "parameters complete": the last CTA of the grid (atomic ticket) fences, tells every peer, and waits for every peer's
//            word — so when the kernel completes, (a) every rank has finished READING this rank's gradients (they may be zeroed for
//            the next step) and (b) every owner has finished WRITING this rank's parameters (the next forward may read them).
// The loss (one fp32 per rank after the gradients) is summed by every rank into a local output word.
// Flags are epochs (step count + 1, identical on all ranks, read from device memory: the launch is CUDA-graph capturable);
// every wait is bounded and traps instead of hanging the device.
// ddfa_allreduce_adam_p2p_guarded adds a norm phase for gradient clipping and skipping (below the first kernel).
#include "common.cuh"
#include "grad_guard.cuh"

namespace ddfa {
namespace p2p {

constexpr int kMaxRanks = 16;
struct Peers {
  float *params[kMaxRanks];
  const float *grads[kMaxRanks];
  uint32_t *flags[kMaxRanks];      // per rank: [0, R) phase-1 words, [R, 2R) phase-2 words, written by the rank of that index
};

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// peer gradients: system-scope relaxed load — never served from this SM's L1 (peer lines are L1-cacheable, B300_MICROARCH)
__device__ __forceinline__ float4 ld_sys_f4(const float *p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void wait_epoch(const uint32_t *p, uint32_t epoch) {
  for (uint32_t it = 0; it < (1u << 23); ++it)      // ~10 s of polling: a rank that never arrives ends in a trap, not a hung device
    if ((int32_t)(ld_acquire_sys(p) - epoch) >= 0) return;
  __trap();
}

__global__ void __launch_bounds__(256) allreduce_adam_p2p_kernel(const Peers pp, int rank, int world, float *__restrict__ m,
                                                                 float *__restrict__ v, const int32_t *__restrict__ step_count,
                                                                 int64_t numel, int64_t loss_off, float *__restrict__ loss_out,
                                                                 uint32_t *__restrict__ ticket, float lr, float beta1, float beta2,
                                                                 float eps, float wd, const float *__restrict__ hyper) {
  if (hyper) {      // [lr, beta1, beta2, eps, wd] read at run time (ddfa_allreduce_adam_p2p_hp); same arithmetic as the by-value form
    lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2], eps = hyper[3], wd = hyper[4];
  }
  __shared__ float s_c[2];
  __shared__ int s_last;
  const int32_t t0 = *step_count;
  const uint32_t epoch = (uint32_t)t0 + 1u;
  if (threadIdx.x == 0) {
    const double t = (double)(t0 + 1);
    s_c[0] = (float)((double)lr / (1.0 - pow((double)beta1, t)));   // step_size
    s_c[1] = (float)sqrt(1.0 - pow((double)beta2, t));              // bias_correction2_sqrt
  }
  // ---- phase 1
  __threadfence_system();
  if (blockIdx.x == 0 && threadIdx.x < world) st_release_sys(pp.flags[threadIdx.x] + rank, epoch);
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + threadIdx.x, epoch);
  __syncthreads();
  const float step_size = s_c[0], bc2s = s_c[1];
  // ---- this rank's slice, in 16-byte units (numel is a multiple of 4: the trainer aligns every parameter to 64 elements)
  const int64_t n4 = numel >> 2;
  const int64_t per = (n4 + world - 1) / world;
  const int64_t lo = (int64_t)rank * per, hi = min(n4, lo + per);
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = 0; p < world; ++p) f4_add(g, ld_sys_f4(pp.grads[p] + 4 * i));     // rank order: the same sum on every run
    float4 w = *reinterpret_cast<const float4 *>(pp.params[rank] + 4 * i);
    float4 mi = *reinterpret_cast<const float4 *>(m + 4 * i), vi = *reinterpret_cast<const float4 *>(v + 4 * i);
#define DDFA_ADAM1(f)                                        \
  {                                                          \
    const float gi = fmaf(wd, w.f, g.f);                     \
    mi.f = fmaf(beta1, mi.f, (1.f - beta1) * gi);            \
    vi.f = fmaf(beta2, vi.f, (1.f - beta2) * gi * gi);       \
    w.f = w.f - step_size * (mi.f / (sqrtf(vi.f) / bc2s + eps)); \
  }
    DDFA_ADAM1(x) DDFA_ADAM1(y) DDFA_ADAM1(z) DDFA_ADAM1(w)
#undef DDFA_ADAM1
    *reinterpret_cast<float4 *>(m + 4 * i) = mi;
    *reinterpret_cast<float4 *>(v + 4 * i) = vi;
    for (int p = 0; p < world; ++p) *reinterpret_cast<float4 *>(pp.params[p] + 4 * i) = w;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && loss_out) {
    float s = 0.f;
    for (int p = 0; p < world; ++p) {
      float x;
      asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(x) : "l"(pp.grads[p] + loss_off) : "memory");
      s += x;
    }
    *loss_out = s;
  }
  // ---- phase 2
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) *ticket = 0u;
  __threadfence_system();
  if (threadIdx.x < world) st_release_sys(pp.flags[threadIdx.x] + world + rank, epoch);
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + world + threadIdx.x, epoch);
}

// ---- guarded form: gradient-norm clipping and skipping of non-finite steps (grad_guard.cuh) ------------------------------------
// A rank reduces only its own 1/R slice, but the norm needs all of them, so a norm phase sits between phase 1 and the update:
//   norm     every CTA sums the squares of its part of the reduced slice in fp64 (a fixed tree) into a per-CTA partial; the last CTA
//            by ticket adds the partials in CTA order and writes the slice sum into EVERY peer's flag area (slot `rank` of the fp64
//            words), then releases an epoch word there.  Every CTA waits for the R epoch words and adds the R slice sums in RANK
//            order, so norm, coefficient and skip decision are bit-identical on every rank.
//   update   the peer gradients are read again (the same rank-order sum) and Adam runs on g * coef; a skipped step writes no
//            parameter or moment and leaves the step counter alone, but still sums the loss and runs phase 2.
// Epochs come from the launch counter in GuardState, not from the step count: a skipped step does not advance the step count, and
// an epoch that repeats would let the next launch through the barriers unsynchronised.
// Flag words per rank: [0, R) phase 1, [R, 2R) phase 2, [2R, 3R) norm epochs, fp64 slice sums from word kSumWord (8-byte aligned).
constexpr int kSumWord = 64, kGuardFlagWords = kSumWord + 2 * kMaxRanks;     // 96 >= 3 * kMaxRanks
static_assert(kGuardFlagWords == DDFA_P2P_GUARD_FLAG_WORDS && 3 * kMaxRanks <= kSumWord, "guarded flag layout");
constexpr int kMaxCtas = 64;
struct GuardState {
  uint32_t ticket[2];      // norm phase, phase 2: each returns to 0 within the launch
  uint32_t launches;       // launches completed: the next epoch is launches + 1
  uint32_t pad;
  double partial[kMaxCtas];
};

__device__ __forceinline__ void st_relaxed_sys_f64(uint32_t *p, double v) {
  asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ double ld_relaxed_sys_f64(const uint32_t *p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(256) allreduce_adam_p2p_guarded_kernel(const Peers pp, int rank, int world, float *__restrict__ m,
                                                                         float *__restrict__ v, int32_t *__restrict__ step_count,
                                                                         int64_t numel, int64_t loss_off, float *__restrict__ loss_out,
                                                                         GuardState *__restrict__ gs, const float *__restrict__ hyper,
                                                                         const float *__restrict__ max_norm, float *__restrict__ gstate,
                                                                         int32_t *__restrict__ skipped) {
  const float lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2], eps = hyper[3], wd = hyper[4];
  __shared__ float s_c[2];
  __shared__ double s_red[256];
  __shared__ float s_coef;
  __shared__ int s_last, s_skip;
  const int32_t t0 = *step_count;
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t *>(&gs->launches) + 1u;
  if (threadIdx.x == 0) {
    const double t = (double)(t0 + 1);
    s_c[0] = (float)((double)lr / (1.0 - pow((double)beta1, t)));   // step_size
    s_c[1] = (float)sqrt(1.0 - pow((double)beta2, t));              // bias_correction2_sqrt
  }
  // ---- phase 1
  __threadfence_system();
  if (blockIdx.x == 0 && threadIdx.x < world) st_release_sys(pp.flags[threadIdx.x] + rank, epoch);
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + threadIdx.x, epoch);
  __syncthreads();
  const float step_size = s_c[0], bc2s = s_c[1];
  const int64_t n4 = numel >> 2;
  const int64_t per = (n4 + world - 1) / world;
  const int64_t lo = (int64_t)rank * per, hi = min(n4, lo + per);
  // ---- norm: this CTA's part of the reduced slice
  double acc = 0.0;
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = 0; p < world; ++p) f4_add(g, ld_sys_f4(pp.grads[p] + 4 * i));     // rank order, as in the update below
    acc += guard::sq(g.x);
    acc += guard::sq(g.y);
    acc += guard::sq(g.z);
    acc += guard::sq(g.w);
  }
  s_red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    gs->partial[blockIdx.x] = s_red[0];
    __threadfence();
    s_last = (atomicAdd(&gs->ticket[0], 1u) == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (s_last) {      // the slice sum, in CTA order, to every rank
    if (threadIdx.x == 0) {
      gs->ticket[0] = 0u;
      __threadfence();
      double s = 0.0;
      for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(&gs->partial[c]);
      s_red[0] = s;
    }
    __syncthreads();
    if (threadIdx.x < world) {
      st_relaxed_sys_f64(pp.flags[threadIdx.x] + kSumWord + 2 * rank, s_red[0]);
      st_release_sys(pp.flags[threadIdx.x] + 2 * world + rank, epoch);       // orders the store above before the epoch
    }
  }
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + 2 * world + threadIdx.x, epoch);
  __syncthreads();
  if (threadIdx.x == 0) {
    double total = 0.0;
    for (int p = 0; p < world; ++p) total += ld_relaxed_sys_f64(pp.flags[rank] + kSumWord + 2 * p);
    float norm, coef;
    bool nonfinite;
    guard::finish(total, max_norm, &norm, &coef, &nonfinite);
    s_coef = coef;
    s_skip = (skipped != nullptr && nonfinite) ? 1 : 0;
    if (blockIdx.x == 0) {
      gstate[guard::kNorm] = norm;
      gstate[guard::kCoef] = coef;
      gstate[guard::kNonFinite] = nonfinite ? 1.f : 0.f;
    }
  }
  __syncthreads();
  // ---- update (allreduce_adam_p2p_kernel's arithmetic on g * coef; coef == 1 leaves g bit-unchanged)
  const float coef = s_coef;
  if (!s_skip) {
    for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int p = 0; p < world; ++p) f4_add(g, ld_sys_f4(pp.grads[p] + 4 * i));
      float4 w = *reinterpret_cast<const float4 *>(pp.params[rank] + 4 * i);
      float4 mi = *reinterpret_cast<const float4 *>(m + 4 * i), vi = *reinterpret_cast<const float4 *>(v + 4 * i);
#define DDFA_ADAM1(f)                                        \
  {                                                          \
    const float gi = fmaf(wd, w.f, g.f * coef);              \
    mi.f = fmaf(beta1, mi.f, (1.f - beta1) * gi);            \
    vi.f = fmaf(beta2, vi.f, (1.f - beta2) * gi * gi);       \
    w.f = w.f - step_size * (mi.f / (sqrtf(vi.f) / bc2s + eps)); \
  }
      DDFA_ADAM1(x) DDFA_ADAM1(y) DDFA_ADAM1(z) DDFA_ADAM1(w)
#undef DDFA_ADAM1
      *reinterpret_cast<float4 *>(m + 4 * i) = mi;
      *reinterpret_cast<float4 *>(v + 4 * i) = vi;
      for (int p = 0; p < world; ++p) *reinterpret_cast<float4 *>(pp.params[p] + 4 * i) = w;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && loss_out) {
    float s = 0.f;
    for (int p = 0; p < world; ++p) {
      float x;
      asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(x) : "l"(pp.grads[p] + loss_off) : "memory");
      s += x;
    }
    *loss_out = s;
  }
  // ---- phase 2; the last CTA also advances the counters (every CTA has read them by now)
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&gs->ticket[1], 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) {
    gs->ticket[1] = 0u;
    gs->launches = epoch;
    if (s_skip)
      *skipped += 1;
    else
      *step_count = t0 + 1;
  }
  __threadfence_system();
  if (threadIdx.x < world) st_release_sys(pp.flags[threadIdx.x] + world + rank, epoch);
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + world + threadIdx.x, epoch);
}

}  // namespace p2p
}  // namespace ddfa

namespace ddfa {
namespace p2p {

static int fill_peers(Peers &pp, void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int world) {
  for (int p = 0; p < world; ++p) {
    DDFA_REQUIRE(peer_params[p] && peer_grads[p] && peer_flags[p] && aligned16(peer_params[p]) && aligned16(peer_grads[p]) &&
                     aligned16(peer_flags[p]),
                 "ddfa_allreduce_adam_p2p_guarded: peer %d pointer NULL or unaligned", p);
    pp.params[p] = static_cast<float *>(peer_params[p]);
    pp.grads[p] = static_cast<const float *>(peer_grads[p]);
    pp.flags[p] = static_cast<uint32_t *>(peer_flags[p]);
  }
  return DDFA_OK;
}

static int launch(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank, int32_t world,
                  float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel, int64_t loss_offset, float *loss_out,
                  uint32_t *ticket, float lr, float beta1, float beta2, float eps, float weight_decay, const float *hyper,
                  void *stream_) {
  DDFA_REQUIRE(world >= 1 && world <= p2p::kMaxRanks && rank >= 0 && rank < world, "ddfa_allreduce_adam_p2p: rank %d / world %d (max %d ranks)", rank,
               world, p2p::kMaxRanks);
  DDFA_REQUIRE(numel >= 0 && numel % 4 == 0, "ddfa_allreduce_adam_p2p: numel (%lld) must be a multiple of 4", (long long)numel);
  DDFA_REQUIRE(peer_params && peer_grads && peer_flags && exp_avg && exp_avg_sq && step_count && ticket, "ddfa_allreduce_adam_p2p: NULL pointer");
  p2p::Peers pp = {};
  for (int p = 0; p < world; ++p) {
    DDFA_REQUIRE(peer_params[p] && peer_grads[p] && peer_flags[p] && aligned16(peer_params[p]) && aligned16(peer_grads[p]),
                 "ddfa_allreduce_adam_p2p: peer %d pointer NULL or unaligned", p);
    pp.params[p] = static_cast<float *>(peer_params[p]);
    pp.grads[p] = static_cast<const float *>(peer_grads[p]);
    pp.flags[p] = static_cast<uint32_t *>(peer_flags[p]);
  }
  cudaStream_t stream = as_stream(stream_);
  const int64_t per = ((numel >> 2) + world - 1) / world;
  int blocks = (int)((per + 255) / 256);
  if (blocks < 1) blocks = 1;
  if (blocks > 64) blocks = 64;        // all CTAs must be co-resident: they spin on flags (64 x 256 threads fit any idle H100)
  p2p::allreduce_adam_p2p_kernel<<<blocks, 256, 0, stream>>>(pp, rank, world, exp_avg, exp_avg_sq, step_count, numel, loss_offset, loss_out, ticket,
                                                             lr, beta1, beta2, eps, weight_decay, hyper);
  DDFA_CHECK_LAUNCH("allreduce_adam_p2p_kernel");
  return adam_step_inc_launch(step_count, stream);
}

}  // namespace p2p
}  // namespace ddfa

extern "C" int ddfa_allreduce_adam_p2p(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank,
                                       int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                                       int64_t loss_offset, float *loss_out, uint32_t *ticket, float lr, float beta1, float beta2,
                                       float eps, float weight_decay, void *stream_) {
  return ddfa::p2p::launch(peer_params, peer_grads, peer_flags, rank, world, exp_avg, exp_avg_sq, step_count, numel, loss_offset, loss_out,
                           ticket, lr, beta1, beta2, eps, weight_decay, nullptr, stream_);
}

extern "C" int ddfa_allreduce_adam_p2p_hp(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank,
                                          int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                                          int64_t loss_offset, float *loss_out, uint32_t *ticket, const float *hyper, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(hyper, "ddfa_allreduce_adam_p2p_hp: NULL hyperparameter pointer");
  return p2p::launch(peer_params, peer_grads, peer_flags, rank, world, exp_avg, exp_avg_sq, step_count, numel, loss_offset, loss_out, ticket,
                     0.f, 0.f, 0.f, 0.f, 0.f, hyper, stream_);
}

extern "C" size_t ddfa_p2p_guard_state_bytes(void) { return sizeof(ddfa::p2p::GuardState); }

extern "C" int ddfa_allreduce_adam_p2p_guarded(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                                               int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                                               int64_t numel, int64_t loss_offset, float *loss_out, const float *hyper,
                                               const float *max_norm, float *gstate, int32_t *skipped, void *guard_state,
                                               void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(world >= 1 && world <= p2p::kMaxRanks && rank >= 0 && rank < world, "ddfa_allreduce_adam_p2p_guarded: rank %d / world %d (max %d ranks)",
               rank, world, p2p::kMaxRanks);
  DDFA_REQUIRE(numel >= 0 && numel % 4 == 0, "ddfa_allreduce_adam_p2p_guarded: numel (%lld) must be a multiple of 4", (long long)numel);
  DDFA_REQUIRE(peer_params && peer_grads && peer_flags && exp_avg && exp_avg_sq && step_count && hyper && gstate && guard_state,
               "ddfa_allreduce_adam_p2p_guarded: NULL pointer");
  DDFA_REQUIRE(aligned16(guard_state), "ddfa_allreduce_adam_p2p_guarded: guard_state must be 16-byte aligned");
  p2p::Peers pp = {};
  const int rc = p2p::fill_peers(pp, peer_params, peer_grads, peer_flags, world);
  if (rc != DDFA_OK) return rc;
  cudaStream_t stream = as_stream(stream_);
  const int64_t per = ((numel >> 2) + world - 1) / world;
  int blocks = (int)((per + 255) / 256);
  if (blocks < 1) blocks = 1;
  if (blocks > p2p::kMaxCtas) blocks = p2p::kMaxCtas;     // co-resident (they spin on flags), and one partial slot each
  p2p::allreduce_adam_p2p_guarded_kernel<<<blocks, 256, 0, stream>>>(pp, rank, world, exp_avg, exp_avg_sq, step_count, numel, loss_offset,
                                                                     loss_out, static_cast<p2p::GuardState *>(guard_state), hyper,
                                                                     max_norm, gstate, skipped);
  DDFA_CHECK_LAUNCH("allreduce_adam_p2p_guarded_kernel");
  return DDFA_OK;
}
