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
// Flags are epochs (identical on all ranks, read from device memory: the launch is CUDA-graph capturable); every wait is bounded
// and traps instead of hanging the device.
//
// ddfa_allreduce_adam_p2p[_hp] and ddfa_allreduce_adam_p2p_guarded run one kernel, allreduce_adam_p2p_kernel<Guarded, Grouped>;
// the _groups forms (Grouped) update only the parts of the slice inside a list of [begin, end, group] ranges, each with its
// parameter group's row of a device table (coupled Adam or decoupled AdamW, adam.cuh) and bias correction.  The norm of the
// guarded form covers the whole slice either way.
// The guarded form (gradient clipping and skipping of non-finite steps, adam.cuh) differs in four places:
//   norm     a rank reduces only its own 1/R slice, but the norm needs all of them, so a norm phase sits between phase 1 and the
//            update: every CTA sums the squares of its part of the reduced slice in fp64 (a fixed tree) into a per-CTA partial;
//            the last CTA by ticket adds the partials in CTA order and writes the slice sum into EVERY peer's flag area (slot
//            `rank` of the fp64 words), then releases an epoch word there.  Every CTA waits for the R epoch words and adds the R
//            slice sums in RANK order, so norm, coefficient and skip decision are bit-identical on every rank.  The update then
//            reads the peer gradients again (the same rank-order sum) and runs on g * coef; a skipped step writes no parameter
//            or moment, but still sums the loss and runs phase 2.
//   epochs   step count + 1 unguarded.  Guarded, the launch counter in GuardState + 1: a skipped step does not advance the step
//            count, and an epoch that repeats would let the next launch through the barriers unsynchronised.
//   tickets  the caller's ticket word unguarded; GuardState's two tickets (norm phase, phase 2) guarded.
//   counters unguarded, a separate 1-thread launch increments the step count; guarded, the last CTA of phase 2 advances the
//            launch counter and the step or the skip counter (every CTA has read them by then).
// Flag words per rank: [0, R) phase 1, [R, 2R) phase 2; guarded also [2R, 3R) norm epochs, fp64 slice sums from word kSumWord.
#include "common.cuh"
#include "adam.cuh"

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

// Flag words per rank as listed above; the fp64 slice sums are 8-byte aligned.
constexpr int kSumWord = 64, kGuardFlagWords = kSumWord + 2 * kMaxRanks;     // 96 >= 3 * kMaxRanks
static_assert(kGuardFlagWords == DDFA_P2P_GUARD_FLAG_WORDS && 3 * kMaxRanks <= kSumWord, "guarded flag layout");
constexpr int kMaxCtas = 64;     // all CTAs must be co-resident: they spin on flags (64 x 256 threads fit any idle H100)
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

// ---- the protocol's steps, shared by both forms of the kernel

// phase 1 "gradients complete": CTA 0 tells every peer, every CTA waits for every peer
__device__ __forceinline__ void phase1(const Peers &pp, int rank, int world, uint32_t epoch) {
  __threadfence_system();
  if (blockIdx.x == 0 && threadIdx.x < world) st_release_sys(pp.flags[threadIdx.x] + rank, epoch);
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + threadIdx.x, epoch);
  __syncthreads();
}

// the reduced gradient of 16-byte unit i, summed in rank order: the same sum on every run and in every pass
__device__ __forceinline__ float4 reduced_grad(const Peers &pp, int world, int64_t i) {
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = 0; p < world; ++p) f4_add(g, ld_sys_f4(pp.grads[p] + 4 * i));
  return g;
}

// Adam on this rank's units [lo, hi) (guarded: on g * coef); the new parameters go to every rank.  H: adam::Hyper (one coupled
// group) or adam::Group (a row of the group table).
template <bool Guarded, typename H>
__device__ __forceinline__ void update_slice(const Peers &pp, int rank, int world, float *__restrict__ m, float *__restrict__ v, int64_t lo,
                                             int64_t hi, const H &h, const adam::Bias &c, float coef) {
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    float4 g = reduced_grad(pp, world, i);
    if constexpr (Guarded) g = make_float4(g.x * coef, g.y * coef, g.z * coef, g.w * coef);
    float4 w = *reinterpret_cast<const float4 *>(pp.params[rank] + 4 * i);
    float4 mi = *reinterpret_cast<const float4 *>(m + 4 * i), vi = *reinterpret_cast<const float4 *>(v + 4 * i);
    adam::update(g, w, mi, vi, h, c);
    *reinterpret_cast<float4 *>(m + 4 * i) = mi;
    *reinterpret_cast<float4 *>(v + 4 * i) = vi;
    for (int p = 0; p < world; ++p) *reinterpret_cast<float4 *>(pp.params[p] + 4 * i) = w;
  }
}

// Parameter groups: this rank's units [lo, hi) intersected with every [begin, end, group] range (bounds multiples of 4), each
// with its group's row and bias correction (shared memory); units outside every range are neither read nor written.
template <bool Guarded>
__device__ __forceinline__ void update_slice_groups(const Peers &pp, int rank, int world, float *__restrict__ m, float *__restrict__ v,
                                                    int64_t lo, int64_t hi, const int64_t *__restrict__ ranges, int32_t num_ranges,
                                                    int32_t num_groups, const adam::Group *s_g, const adam::Bias *s_c, float coef) {
  for (int32_t r = 0; r < num_ranges; ++r) {
    const int64_t grp = ranges[3 * r + 2];
    if (grp < 0 || grp >= num_groups) continue;
    const int64_t a = max(lo, ranges[3 * r] >> 2), b = min(hi, ranges[3 * r + 1] >> 2);
    if (a < b) update_slice<Guarded>(pp, rank, world, m, v, a, b, s_g[grp], s_c[grp], coef);
  }
}

// the loss words of all ranks, added in rank order into the local word
__device__ __forceinline__ void sum_loss(const Peers &pp, int world, int64_t loss_off, float *loss_out) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && loss_out) {
    float s = 0.f;
    for (int p = 0; p < world; ++p) {
      float x;
      asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(x) : "l"(pp.grads[p] + loss_off) : "memory");
      s += x;
    }
    *loss_out = s;
  }
}

// phase 2 "parameters complete": every CTA but the last by ticket returns; the last resets the ticket, runs last_cta() on thread
// 0 (every other CTA has finished reading the counters by then), tells every peer and waits for every peer
template <typename LastCta>
__device__ __forceinline__ void phase2(const Peers &pp, int rank, int world, uint32_t epoch, uint32_t *ticket, int &s_last,
                                       LastCta last_cta) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) {
    *ticket = 0u;
    last_cta();
  }
  __threadfence_system();
  if (threadIdx.x < world) st_release_sys(pp.flags[threadIdx.x] + world + rank, epoch);
  if (threadIdx.x < world) wait_epoch(pp.flags[rank] + world + threadIdx.x, epoch);
}

// guarded: the norm of the reduced gradients over all ranks (see the top of the file) -> gstate, *coef, *skip (thread 0)
__device__ __forceinline__ void norm_phase(const Peers &pp, int rank, int world, uint32_t epoch, int64_t lo, int64_t hi,
                                          GuardState *__restrict__ gs, const float *__restrict__ max_norm, float *__restrict__ gstate,
                                          const int32_t *skipped, int &s_last, float *coef, int *skip) {
  __shared__ double s_red[256];
  double acc = 0.0;
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 g = reduced_grad(pp, world, i);
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
    float norm, c;
    bool nonfinite;
    guard::finish(total, max_norm, &norm, &c, &nonfinite);
    *coef = c;
    *skip = (skipped != nullptr && nonfinite) ? 1 : 0;
    if (blockIdx.x == 0) {
      gstate[guard::kNorm] = norm;
      gstate[guard::kCoef] = c;
      gstate[guard::kNonFinite] = nonfinite ? 1.f : 0.f;
    }
  }
  __syncthreads();
}

// Unguarded: ticket is the caller's word, gs .. skipped are NULL.  Guarded: ticket is NULL.  Grouped: h / hyper are unused and
// ranges / table (num_groups rows) select each element's group; otherwise ranges and table are NULL.
template <bool Guarded, bool Grouped>
__global__ void __launch_bounds__(256) allreduce_adam_p2p_kernel(const Peers pp, int rank, int world, float *__restrict__ m,
                                                                 float *__restrict__ v, int32_t *__restrict__ step_count, int64_t numel,
                                                                 int64_t loss_off, float *__restrict__ loss_out, uint32_t *__restrict__ ticket,
                                                                 adam::Hyper h, const float *__restrict__ hyper, GuardState *__restrict__ gs,
                                                                 const float *__restrict__ max_norm, float *__restrict__ gstate,
                                                                 int32_t *__restrict__ skipped, const int64_t *__restrict__ ranges,
                                                                 int32_t num_ranges, const float *__restrict__ table, int32_t num_groups) {
  __shared__ adam::Bias s_c;
  __shared__ adam::Group s_grp[Grouped ? adam::kMaxGroups : 1];
  __shared__ adam::Bias s_grp_c[Grouped ? adam::kMaxGroups : 1];
  __shared__ float s_coef;
  __shared__ int s_last, s_skip;
  const int32_t t0 = *step_count;
  const uint32_t epoch = (Guarded ? *reinterpret_cast<volatile uint32_t *>(&gs->launches) : (uint32_t)t0) + 1u;
  if constexpr (Grouped) {
    adam::load_groups(table, num_groups, t0, s_grp, s_grp_c);      // phase1 ends with __syncthreads
  } else {
    h = adam::load(h, hyper);
    if (threadIdx.x == 0) s_c = adam::bias_correction(h.lr, h.beta1, h.beta2, t0);
  }
  phase1(pp, rank, world, epoch);
  const adam::Bias c = s_c;
  // this rank's slice, in 16-byte units (numel is a multiple of 4: the trainer aligns every parameter to 64 elements)
  const int64_t n4 = numel >> 2;
  const int64_t per = (n4 + world - 1) / world;
  const int64_t lo = (int64_t)rank * per, hi = min(n4, lo + per);
  if constexpr (Guarded) {
    norm_phase(pp, rank, world, epoch, lo, hi, gs, max_norm, gstate, skipped, s_last, &s_coef, &s_skip);
    if (!s_skip) {
      if constexpr (Grouped)
        update_slice_groups<true>(pp, rank, world, m, v, lo, hi, ranges, num_ranges, num_groups, s_grp, s_grp_c, s_coef);
      else
        update_slice<true>(pp, rank, world, m, v, lo, hi, h, c, s_coef);
    }
  } else if constexpr (Grouped) {
    update_slice_groups<false>(pp, rank, world, m, v, lo, hi, ranges, num_ranges, num_groups, s_grp, s_grp_c, 1.f);
  } else {
    update_slice<false>(pp, rank, world, m, v, lo, hi, h, c, 1.f);
  }
  sum_loss(pp, world, loss_off, loss_out);
  if constexpr (Guarded) {
    phase2(pp, rank, world, epoch, &gs->ticket[1], s_last, [&] {
      gs->launches = epoch;
      if (s_skip)
        *skipped += 1;
      else
        *step_count = t0 + 1;
    });
  } else {
    phase2(pp, rank, world, epoch, ticket, s_last, [] {});
  }
}

// Argument checks (`name` is the entry point), Peers, the grid, the launch.  Unguarded, the step-count increment follows as a
// launch of its own; guarded, the kernel advances the counters itself.
template <bool Guarded, bool Grouped = false>
static int launch(const char *name, void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank,
                  int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel, int64_t loss_offset, float *loss_out,
                  uint32_t *ticket, adam::Hyper h, const float *hyper, void *guard_state, const float *max_norm, float *gstate,
                  int32_t *skipped, void *stream_, const int64_t *ranges = nullptr, int32_t num_ranges = 0, const float *table = nullptr,
                  int32_t num_groups = 0) {
  DDFA_REQUIRE(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world, "%s: rank %d / world %d (max %d ranks)", name, rank, world,
               kMaxRanks);
  DDFA_REQUIRE(numel >= 0 && numel % 4 == 0, "%s: numel (%lld) must be a multiple of 4", name, (long long)numel);
  DDFA_REQUIRE(peer_params && peer_grads && peer_flags && exp_avg && exp_avg_sq && step_count &&
                   (Guarded ? (Grouped || hyper) && gstate && guard_state : ticket != nullptr),
               "%s: NULL pointer", name);
  if constexpr (Grouped) {
    DDFA_REQUIRE(num_ranges >= 0 && num_groups >= 1 && num_groups <= adam::kMaxGroups,
                 "%s: num_ranges (%d) must be >= 0 and num_groups (%d) in [1, %d]", name, num_ranges, num_groups, adam::kMaxGroups);
    DDFA_REQUIRE(table && (ranges || num_ranges == 0), "%s: NULL pointer", name);
  }
  DDFA_REQUIRE(!Guarded || aligned16(guard_state), "%s: guard_state must be 16-byte aligned", name);
  Peers pp = {};
  for (int p = 0; p < world; ++p) {
    // the guarded kernel's fp64 slice sums live in the flag words
    DDFA_REQUIRE(peer_params[p] && peer_grads[p] && peer_flags[p] && aligned16(peer_params[p]) && aligned16(peer_grads[p]) &&
                     (!Guarded || aligned16(peer_flags[p])),
                 "%s: peer %d pointer NULL or unaligned", name, p);
    pp.params[p] = static_cast<float *>(peer_params[p]);
    pp.grads[p] = static_cast<const float *>(peer_grads[p]);
    pp.flags[p] = static_cast<uint32_t *>(peer_flags[p]);
  }
  cudaStream_t stream = as_stream(stream_);
  const int64_t per = ((numel >> 2) + world - 1) / world;
  int blocks = (int)((per + 255) / 256);
  if (blocks < 1) blocks = 1;
  if (blocks > kMaxCtas) blocks = kMaxCtas;     // co-resident, and one partial slot each
  allreduce_adam_p2p_kernel<Guarded, Grouped><<<blocks, 256, 0, stream>>>(pp, rank, world, exp_avg, exp_avg_sq, step_count, numel, loss_offset,
                                                                          loss_out, ticket, h, hyper, static_cast<GuardState *>(guard_state),
                                                                          max_norm, gstate, skipped, ranges, num_ranges, table, num_groups);
  DDFA_CHECK_LAUNCH("allreduce_adam_p2p_kernel");
  return Guarded ? DDFA_OK : adam_step_inc_launch(step_count, nullptr, nullptr, stream);
}

}  // namespace p2p
}  // namespace ddfa

extern "C" int ddfa_allreduce_adam_p2p(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank,
                                       int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                                       int64_t loss_offset, float *loss_out, uint32_t *ticket, float lr, float beta1, float beta2,
                                       float eps, float weight_decay, void *stream_) {
  using namespace ddfa;
  return p2p::launch<false>("ddfa_allreduce_adam_p2p", peer_params, peer_grads, peer_flags, rank, world, exp_avg, exp_avg_sq, step_count,
                            numel, loss_offset, loss_out, ticket, adam::Hyper{lr, beta1, beta2, eps, weight_decay}, nullptr, nullptr,
                            nullptr, nullptr, nullptr, stream_);
}

extern "C" int ddfa_allreduce_adam_p2p_hp(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank,
                                          int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                                          int64_t loss_offset, float *loss_out, uint32_t *ticket, const float *hyper, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(hyper, "ddfa_allreduce_adam_p2p_hp: NULL hyperparameter pointer");
  return p2p::launch<false>("ddfa_allreduce_adam_p2p_hp", peer_params, peer_grads, peer_flags, rank, world, exp_avg, exp_avg_sq, step_count,
                            numel, loss_offset, loss_out, ticket, adam::Hyper{}, hyper, nullptr, nullptr, nullptr, nullptr, stream_);
}

extern "C" size_t ddfa_p2p_guard_state_bytes(void) { return sizeof(ddfa::p2p::GuardState); }

extern "C" int ddfa_allreduce_adam_p2p_guarded(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                                               int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                                               int64_t numel, int64_t loss_offset, float *loss_out, const float *hyper,
                                               const float *max_norm, float *gstate, int32_t *skipped, void *guard_state,
                                               void *stream_) {
  using namespace ddfa;
  return p2p::launch<true>("ddfa_allreduce_adam_p2p_guarded", peer_params, peer_grads, peer_flags, rank, world, exp_avg, exp_avg_sq,
                           step_count, numel, loss_offset, loss_out, nullptr, adam::Hyper{}, hyper, guard_state, max_norm, gstate, skipped,
                           stream_);
}

// Parameter groups (torch.optim.AdamW / Adam with several param_groups): the protocol of ddfa_allreduce_adam_p2p_hp and
// ddfa_allreduce_adam_p2p_guarded, with Adam on the intersection of this rank's slice with the [begin, end, group] ranges.
extern "C" int ddfa_allreduce_adam_p2p_groups(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags, int32_t rank,
                                              int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count, int64_t numel,
                                              int64_t loss_offset, float *loss_out, uint32_t *ticket, const int64_t *ranges, int32_t num_ranges,
                                              const float *groups, int32_t num_groups, void *stream_) {
  using namespace ddfa;
  return p2p::launch<false, true>("ddfa_allreduce_adam_p2p_groups", peer_params, peer_grads, peer_flags, rank, world, exp_avg, exp_avg_sq,
                                  step_count, numel, loss_offset, loss_out, ticket, adam::Hyper{}, nullptr, nullptr, nullptr, nullptr, nullptr,
                                  stream_, ranges, num_ranges, groups, num_groups);
}

extern "C" int ddfa_allreduce_adam_p2p_groups_guarded(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                                                      int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                                                      int64_t numel, int64_t loss_offset, float *loss_out, const int64_t *ranges,
                                                      int32_t num_ranges, const float *groups, int32_t num_groups, const float *max_norm,
                                                      float *gstate, int32_t *skipped, void *guard_state, void *stream_) {
  using namespace ddfa;
  return p2p::launch<true, true>("ddfa_allreduce_adam_p2p_groups_guarded", peer_params, peer_grads, peer_flags, rank, world, exp_avg,
                                 exp_avg_sq, step_count, numel, loss_offset, loss_out, nullptr, adam::Hyper{}, nullptr, guard_state, max_norm,
                                 gstate, skipped, stream_, ranges, num_ranges, groups, num_groups);
}
