// Shared helpers for libddfa_b200.so (sm_90a only: NVIDIA H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ddfa_b200.h"

namespace ddfa {

void set_error(const char *fmt, ...);
void count_launch();  // abi.cu: process-wide counter of kernel launches issued by this library

inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

#define DDFA_REQUIRE(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ddfa::set_error(__VA_ARGS__);        \
      return DDFA_ERR_INVALID_ARG;         \
    }                                      \
  } while (0)

#define DDFA_CHECK_LAUNCH(name)                                                        \
  do {                                                                                 \
    cudaError_t e__ = cudaGetLastError();                                              \
    if (e__ != cudaSuccess) {                                                          \
      ddfa::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));         \
      return DDFA_ERR_CUDA;                                                            \
    }                                                                                  \
    ddfa::count_launch();                                                              \
  } while (0)

#define DDFA_CUDA(call)                                                                \
  do {                                                                                 \
    cudaError_t e__ = (call);                                                          \
    if (e__ != cudaSuccess) {                                                          \
      ddfa::set_error("%s failed: %s", #call, cudaGetErrorString(e__));                \
      return DDFA_ERR_CUDA;                                                            \
    }                                                                                  \
  } while (0)

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------------------
// The per-step kernels form a chain in one stream.  Launched with the programmatic-serialization attribute, kernel i+1's CTAs
// may start as soon as every CTA of kernel i has called pdl_launch_dependents() and an SM has room — i.e. in kernel i's tail
// (the persistent GEMM kernels leave part of the SMs idle at the end, when the tiles do not divide evenly over the CTA groups) —
// run their prologue (barrier init, the weight copy into shared memory) and then block in pdl_wait() until kernel i has completed and its
// writes are visible.  Rules for every kernel launched this way:
//   * nothing is written before pdl_wait();
//   * the only global data read before pdl_wait() are the packed weights of the pass;
//   * EVERY global load of a chain kernel is ld.global.cg (L2 only), before and after the wait: between two kernels chained
//     this way the SM's L1 is not invalidated, so an L1-cached load (ld.global.nc / __ldg, or a default ld.global) can return
//     a line fetched before an earlier kernel rewrote that address.  Measured: with gather_image AND gru_fwd3 chained and
//     __ldg loads, a training run over per-shape static input buffers read the previous batch's CSR arrays
//     (tests/test_parity_gpu.py::test_fused_trainer_cuda_graph_paths_match_eager caught it; either kernel alone passed);
//   * the kernel that follows a weight-packing kernel is launched normally (chain_break()), so the packed weights are
//     complete and flushed before any chain kernel can start its prologue.
// Both instructions are no-ops in a normal launch.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
int pdl_mask();       // abi.cu: DDFA_TUNE_PDL_MASK — bit mask of the kernels launched programmatically (1 gather_image, 2 gru_fwd3,
                      // 4 the head of the backward step: bwd_step_fused_kernel or gate_bwd_image_kernel, 8 dgrad3 after gate_bwd_image)
int gather_variant(); // abi.cu: DDFA_TUNE_GATHER_VARIANT
int gather_src_groups();   // abi.cu: DDFA_TUNE_GATHER_SRC_GROUPS — row groups per warp of the image->image gather (0 = by size)
int gate_bwd_tma();   // abi.cu: DDFA_TUNE_GATE_BWD_TMA — gate backward fused into dgrad (packed saved state)
bool deterministic(); // abi.cu: DDFA_TUNE_DETERMINISTIC — reductions summed in a fixed order (no float atomics)
void chain_break();  // abi.cu: the next launch_chain() on this thread is a normal (fully serialised) launch
bool chain_take_break();

// cluster_x > 1: the grid is launched as thread-block clusters of that many CTAs along x
template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain_cluster(int which, int cluster_x, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                        cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = (unsigned)cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  const bool brk = chain_take_break();
  if ((pdl_mask() & which) && !brk) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(int which, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  return launch_chain_cluster(which, 1, kernel, grid, block, smem, stream, args...);
}

// loss_adam.cu: the 1-thread step-count increment after the Adam update (gstate / skipped: the guard's skip rule, or NULL)
int adam_step_inc_launch(int32_t *step_count, const float *gstate, int32_t *skipped, cudaStream_t stream);

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

constexpr int kNumSMs = 132;  // H100 SXM

// sgemm.cu — SIMT fp32 GEMM, C = alpha*op(A)op(B) + beta*C (row-major)
int sgemm(int ta, int tb, int M, int N, int K, float alpha, const float *A, int lda, const float *B, int ldb,
          float beta, float *C, int ldc, int split_k, cudaStream_t stream);
// C[M,N] += alpha * A^T B with K split over split_k slices whose products go to part (sgemm_splitk_ordered_slices(K, split_k) x M x N
// floats) and are added to C in slice order: the deterministic form of a split-K accumulation
int sgemm_splitk_ordered_slices(int K, int split_k);
int sgemm_splitk_ordered(int M, int N, int K, float alpha, const float *A, int lda, const float *B, int ldb, float *C, int ldc,
                         int split_k, float *part, cudaStream_t stream);
// csr_build.cu — in-place inclusive scan of a[1..n] (a[0] stays 0) for one or two int32 arrays (a1 may be NULL); s0 / s1 hold
// the block sums of the multi-CTA form, scan_block_sums_len(n) ints each (NULL: single-CTA form)
int32_t scan_block_sums_len(int32_t n);
int scan_counts(int32_t *a0, int32_t *a1, int32_t n, int32_t *s0, int32_t *s1, cudaStream_t stream);
// gru_tc_fwd3.cu — tensor-core engine, forward (D == 128): activation images
size_t act_image_bytes(int64_t n);
int act_to_image(const float *x, int32_t N, void *image, cudaStream_t stream);
int act_to_image(const float *x, int32_t N, int32_t D, void *image, cudaStream_t stream);   // D columns, D % 64 == 0 (tc_common.cuh: image_offset_w)
// gru_tc_wide.cu — tensor-core GEMMs of the GRU step at the wide widths (192 <= D <= 512, D % 64 == 0), SIMT data flow around them.
// Both step workspaces start with the W' and Whh operand images (gru_tcw_weights_bytes(D), written by gru_tcw_prepare); the
// scratch is the images of the step's GEMM operands (and, backward, the split-K slices of the weight gradient).
bool gru_tcw_width(int32_t D);
size_t gru_tcw_weights_bytes(int32_t D);
size_t gru_tcw_fwd_scratch_bytes(int32_t N, int32_t D);
size_t gru_tcw_bwd_scratch_bytes(int32_t N, int32_t D);
int gru_tcw_prepare(const float *w_fold, const float *w_hh, int32_t D, void *weights, cudaStream_t stream);
// gi = s W'^T, gh = h Whh^T   ([N, 3D] fp32)
int gru_tcw_fwd_gemms(const float *s, const float *h, int32_t N, int32_t D, const void *weights, void *scratch, float *gi, float *gh,
                      cudaStream_t stream);
// ds = dgi W', dh += dgh Whh, dw_fold += dgi^T s, dw_hh += dgh^T h   (weight gradients: split-K slices added in slice order)
int gru_tcw_bwd_gemms(const float *dgi, const float *dgh, const float *s, const float *h, int32_t N, int32_t D, const void *weights,
                      void *scratch, float *ds, float *dh, float *dw_fold, float *dw_hh, cudaStream_t stream);
// gru_tc_fwd3.cu — forward, weights resident in shared memory (wgmma)
size_t gru_tc3_packed_bytes();
int gru_tc3_prepare(const float *w_fold, const float *b_fold, const float *b_ih, const float *w_hh, const float *b_hh, void *packed,
                    cudaStream_t stream);
int gru_tc3_step_fwd(const void *s_img, const void *h_img, const float *h, const int32_t *indptr, int32_t N, float *h_out,
                     void *h_out_img, float *save_gates, void *save_gates_packed, const void *packed, cudaStream_t stream);
int gru_tc3_trace_enable(int on);   // pipeline timeline of gru_fwd3_kernel (development aid)
int gru_tc3_trace_read(void *host, size_t bytes);
int gru_tc2b_trace_enable(int on);  // pipeline timeline of dgrad3_kernel (value 1) / wgrad_kernel (value 2) — development aid
int gru_tc2b_trace_read(void *host, size_t bytes);
int gru_tc2b_fused_max_clusters(int *out);   // 4-CTA clusters of bwd_step_fused_kernel resident at once on this device
size_t gru_tc2_workspace_bytes();
int gru_tc2_prepare(const float *w_fold, const float *b_fold, const float *b_ih, const float *w_hh, const float *b_hh,
                    void *workspace, size_t workspace_bytes, cudaStream_t stream);
int gru_tc2_step_fwd(const void *s_img, const void *h_img, const float *h, const int32_t *indptr, int32_t N, float *h_out,
                     void *h_out_img, float *save_gates, void *save_gates_packed, const void *workspace, size_t workspace_bytes,
                     cudaStream_t stream);
// gru_tc_bwd.cu — tensor-core engine, backward (gate backward -> q images, dgrad, wgrad)
size_t gru_tc2_bwd_workspace_bytes(int32_t N, int32_t slots);
void *gru_tc2_bwd_s_image_scratch(void *workspace, int32_t N);   // one image inside the workspace for the fp32-s entry point
int gru_tc2_prepare_bwd(const float *w_fold, const float *w_hh, void *workspace, size_t workspace_bytes, cudaStream_t stream);
int gru_tc2_step_bwd(const float *dh_out, const float *ds_in, const int32_t *indptr_t, const int32_t *indices_t, const float *h,
                     const void *h_img_in, const void *s_img, const float *gates, const void *gates_packed, const int32_t *indptr, int32_t N, float *ds, float *dh, float *dw_fold, float *db_fold, float *db_ih,
                     float *dw_hh, float *db_hh, void *workspace, size_t workspace_bytes, int wgrad_mode, cudaStream_t stream);
int gru_tc2_bwd_finish(int32_t N, float *dw_fold, float *dw_hh, void *workspace, size_t workspace_bytes, cudaStream_t stream);
int gru_tc2_bwd_wgrad_batched(const void *const *s_imgs, const void *const *h_imgs, int32_t steps, int32_t N, float *dw_fold,
                              float *dw_hh, void *workspace, size_t workspace_bytes, cudaStream_t stream);

// gather_tma.cu — TMA-staged variants (10: per-row bulk copies, 11: tensor-map gather4) of the D == 128 edge gather
int launch_gather_tma(int variant, const int32_t *indptr, const int32_t *indices, const float *h, int32_t N, float *out, int accumulate,
                      cudaStream_t stream);
int gather_tma_errors();   // bounded-wait failures since load (0 in a healthy run)

__device__ __forceinline__ float4 ldg_nc_f4(const float *p) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}

// L2-only load (ld.global.cg): for kernels of the PDL chain, whose L1 may hold lines from before the predecessor's writes
__device__ __forceinline__ float4 ldg_cg_f4(const float *p) { return __ldcg(reinterpret_cast<const float4 *>(p)); }

// ---- L2 eviction-priority hints (createpolicy + .L2::cache_hint) -----------------------------------------------------------
// The train step moves several GB through a 50 MB L2 per step; what a kernel writes for a consumer many kernels later (the saved
// gates) should not push out what the next kernel needs, and what dies after the next kernel (ds, dh, dh'z) should stay.
// kind: 0 = evict_normal, 1 = evict_first, 2 = evict_last.
__device__ __forceinline__ uint64_t l2_policy(int kind) {
  uint64_t p;
  if (kind == 1) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void st_f32_hint(float *p, float v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_f4_hint(float *p, const float4 &v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_f2_hint(float *p, const float2 &v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1,%2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_u4_hint(void *p, const uint4 &v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ float4 ldg_cg_f4_hint(const float *p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.cg.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ float ldg_cg_f32_hint(const float *p, uint64_t pol) {
  float v;
  asm volatile("ld.global.cg.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_u32_hint(void *p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_u2_hint(void *p, const uint2 &v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.u32 [%0], {%1,%2}, %3;" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol) : "memory");
}
// Predicated forms (`@p st`): a store under `if (cond)` becomes a branch, and a branch per output element splits the unrolled
// epilogue of the forward GRU kernel into basic blocks the scheduler cannot interleave (r03 SASS: three branches + a BRA.DIV per
// element); with the predicate inside the instruction the element bodies are straight-line code.
__device__ __forceinline__ void st_f32_hint_if(bool pred, float *p, float v, uint64_t pol) {
  asm volatile("{\n.reg .pred q;\nsetp.ne.b32 q, %3, 0;\n@q st.global.L2::cache_hint.f32 [%0], %1, %2;\n}" ::"l"(p), "f"(v), "l"(pol), "r"((int)pred) : "memory");
}
__device__ __forceinline__ void st_u32_hint_if(bool pred, void *p, uint32_t v, uint64_t pol) {
  asm volatile("{\n.reg .pred q;\nsetp.ne.b32 q, %3, 0;\n@q st.global.L2::cache_hint.u32 [%0], %1, %2;\n}" ::"l"(p), "r"(v), "l"(pol), "r"((int)pred) : "memory");
}
__device__ __forceinline__ void st_u2_hint_if(bool pred, void *p, const uint2 &v, uint64_t pol) {
  asm volatile("{\n.reg .pred q;\nsetp.ne.b32 q, %4, 0;\n@q st.global.L2::cache_hint.v2.u32 [%0], {%1,%2}, %3;\n}" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol), "r"((int)pred)
               : "memory");
}
// abi.cu: DDFA_TUNE_L2_HINTS bit mask, default 23.  1: saved gates written evict_first; 2: saved activations read evict_first in the
// backward pass; 4: ds / dh / dh'z written evict_last; 8: their last reads evict_first; 16: h' and its image written evict_last;
// 32 / 64: operand tiles of the weight-gradient / dgrad kernels copied evict_first.  Whole-step A/B (one box, profiles/r02l-m):
// 4 alone +1.0 %, 7 +1.3 %, 23 +1.9 % over 0; 8, 32, 64 neutral or negative.
int l2_hints();

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// torch.relu: NaN stays NaN (fmaxf(NaN, 0) is 0, which would hide a non-finite activation from the loss, the gradients and the
// non-finite step guard).  Every other input gives fmaxf's result bit for bit, the sign of a zero included.
__device__ __forceinline__ float relu_nan(float y) { return y != y ? y : fmaxf(y, 0.f); }
// ReLU's backward as torch's threshold_backward: the gradient is dropped where the activation is <= 0, so a NaN activation passes it
__device__ __forceinline__ float relu_grad(float act, float g) { return act <= 0.f ? 0.f : g; }

__device__ __forceinline__ void f4_add(float4 &a, const float4 &b) {
  a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
}
__device__ __forceinline__ void f4_fma(float4 &a, float s, const float4 &b) {
  a.x = fmaf(s, b.x, a.x); a.y = fmaf(s, b.y, a.y); a.z = fmaf(s, b.z, a.z); a.w = fmaf(s, b.w, a.w);
}
__device__ __forceinline__ float f4_dot(const float4 &a, const float4 &b) {
  return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
}

}  // namespace ddfa
