// Error plumbing and library-level queries of the C ABI (include/ddfa_b200.h).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>

#include "common.cuh"

namespace ddfa {
static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

static thread_local char g_err[512] = "";

static thread_local bool g_chain_break = true;
void chain_break() { g_chain_break = true; }
bool chain_take_break() {
  const bool b = g_chain_break;
  g_chain_break = false;
  return b;
}

// Tuning knobs (ddfa_tuning_set / ddfa_tuning_get): compiled-in defaults, no environment reads inside the library; the A/B
// scripts set them through the C ABI.  They select between equivalent launch configurations of the same kernels.
static std::atomic<int> g_tuning[DDFA_TUNE__COUNT] = {
    {23},   // DDFA_TUNE_L2_HINTS: measured best on whole-step A/Bs (profiles/r02l-m): 1 + 2 + 4 + 16
    {15},   // DDFA_TUNE_PDL_MASK: all chain kernels (bit 4: the backward step's first kernel, fused or not; 8: dgrad3 after gate_bwd_image)
    {9},    // DDFA_TUNE_GATHER_VARIANT: r01b sweep — 2 rows/pass, 4 loads in flight, 128-thread CTAs
    {0},    // DDFA_TUNE_FWD_PAIR: reserved, only 0 is accepted (no CTA-pair form of the forward kernel on sm_90a)
    {2},    // DDFA_TUNE_GATE_BWD_TMA: 0 gate_bwd_image + dgrad3; 1 bwd_step_fused_kernel (packed saved state); 2 = 1 + CSR scalars pipelined
    {0},    // DDFA_TUNE_GATHER_SRC_GROUPS: image->image gather, row groups per warp (0 = default = 1; 2 / 4 selectable)
    {0},    // DDFA_TUNE_DETERMINISTIC: 0 float atomics where they are fastest; 1 every reduction in a fixed order
};
bool deterministic() { return g_tuning[DDFA_TUNE_DETERMINISTIC].load(std::memory_order_relaxed) != 0; }
int l2_hints() { return g_tuning[DDFA_TUNE_L2_HINTS].load(std::memory_order_relaxed); }
int pdl_mask() { return g_tuning[DDFA_TUNE_PDL_MASK].load(std::memory_order_relaxed); }
int gather_variant() { return g_tuning[DDFA_TUNE_GATHER_VARIANT].load(std::memory_order_relaxed); }
int gate_bwd_tma() { return g_tuning[DDFA_TUNE_GATE_BWD_TMA].load(std::memory_order_relaxed); }
int gather_src_groups() { return g_tuning[DDFA_TUNE_GATHER_SRC_GROUPS].load(std::memory_order_relaxed); }

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace ddfa

extern "C" {

int ddfa_abi_version(void) { return DDFA_ABI_VERSION; }

const char *ddfa_last_error(void) { return ddfa::g_err; }

int ddfa_engine_available(int engine) {
  if (engine == DDFA_ENGINE_SIMT) return 1;
  if (engine == DDFA_ENGINE_TCGEN05) return 1;
  return 0;
}

int ddfa_tuning_set(int key, int value) {
  DDFA_REQUIRE(key >= 0 && key < DDFA_TUNE__COUNT, "ddfa_tuning_set: unknown key %d", key);
  DDFA_REQUIRE(key != DDFA_TUNE_FWD_PAIR || value == 0, "ddfa_tuning_set: DDFA_TUNE_FWD_PAIR must be 0 (no CTA-pair forward kernel on sm_90a)");
  DDFA_REQUIRE(key != DDFA_TUNE_DETERMINISTIC || value == 0 || value == 1, "ddfa_tuning_set: DDFA_TUNE_DETERMINISTIC must be 0 or 1 (got %d)", value);
  ddfa::g_tuning[key].store(value, std::memory_order_relaxed);
  return DDFA_OK;
}
int ddfa_tuning_get(int key) {
  if (key < 0 || key >= DDFA_TUNE__COUNT) return -1;
  return ddfa::g_tuning[key].load(std::memory_order_relaxed);
}

int ddfa_debug_set(int key, int value) {
  switch (key) {
    case 2: {   // pipeline timeline stamps of the tensor-core kernels: 0 off, 1 = gru_fwd3 + dgrad3 / bwd_step_fused, 2 = gru_fwd3 + wgrad
      int rc = ddfa::gru_tc3_trace_enable(value);
      return rc != DDFA_OK ? rc : ddfa::gru_tc2b_trace_enable(value);
    }
    default: ddfa::set_error("ddfa_debug_set: unknown key %d", key); return DDFA_ERR_INVALID_ARG;
  }
}

int ddfa_debug_read(int key, void *host_out, size_t bytes) {
  DDFA_REQUIRE(host_out != nullptr, "ddfa_debug_read: null output");
  switch (key) {   // [132 CTAs][12 tiles][16 events] int64 SM-clock stamps
    case 2: return ddfa::gru_tc2b_trace_read(host_out, bytes);    // dgrad3_kernel / bwd_step_fused_kernel / wgrad_kernel
    case 3: return ddfa::gru_tc3_trace_read(host_out, bytes);     // gru_fwd3_kernel
    case 4: {                                                     // int32: bounded-wait failures of the TMA-staged gather variants
      DDFA_REQUIRE(bytes >= sizeof(int), "ddfa_debug_read: key 4 needs 4 bytes");
      const int v = ddfa::gather_tma_errors();
      memcpy(host_out, &v, sizeof(int));
      return DDFA_OK;
    }
    case 5: {                                                     // int32: 4-CTA clusters of bwd_step_fused_kernel resident at once
      DDFA_REQUIRE(bytes >= sizeof(int), "ddfa_debug_read: key 5 needs 4 bytes");
      int v = 0;
      const int rc = ddfa::gru_tc2b_fused_max_clusters(&v);
      if (rc != DDFA_OK) return rc;
      memcpy(host_out, &v, sizeof(int));
      return DDFA_OK;
    }
    default: ddfa::set_error("ddfa_debug_read: unknown key %d", key); return DDFA_ERR_INVALID_ARG;
  }
}

long long ddfa_launch_count(void) { return ddfa::g_launches.load(std::memory_order_relaxed); }

int ddfa_device_supported(void) {
  int dev = 0;
  DDFA_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  DDFA_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  DDFA_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  return (major == 9 && minor == 0) ? 1 : 0;      // the code is built for sm_90a only
}

}  // extern "C"
