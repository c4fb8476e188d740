// K3, TMA-staged variants of the CSR edge gather-sum (BASELINE north_star: "TMA staging of per-warp edge neighbourhoods into
// shared memory").  Same contract as gather_sum_kernel (gather.cu), D == 128 fp32 rows of 512 B; replaces DGL's
// update_all(copy_u, sum) inside GatedGraphConv (reference call site DDFA/code_gnn/models/flow_gnn/ggnn.py:95).
//
// A warp owns 4 consecutive destination rows.  Instead of pulling the neighbour rows into registers with ld.global, the warp
// stages its edge neighbourhood in a private shared-memory ring through the TMA unit and sums out of shared memory:
//   variant 10  one 1-D bulk copy per neighbour row   (cp.async.bulk.shared::cluster.global, SASS UBLKCP, 512 B each)
//   variant 11  one tensor-map copy per neighbour row (cp.async.bulk.tensor.2d ... tile, box = one 512 B row of the [N, 128] map)
// Completion is an mbarrier transaction count per 8-row batch, two batches in flight per warp (16 x 512 B = 8 KB of ring per
// warp, 64 KB per 8-warp CTA, 3 CTAs per SM = 192 KB of gathers in flight per SM).  No atomics; summation order = neighbour
// order, as in the register kernel, so the three produce bit-identical sums.
// Selected through ddfa_gather_sum_variant(10 | 11, ...) and measured against the register variants by scripts/gather_bench.py;
// DESIGN.md §3 has the A/B.
#include <cuda.h>
#include <string.h>

#include "tc_common.cuh"

namespace ddfa {
namespace gtma {
using tcc::bulk_g2s;
using tcc::mbar_arrive_expect_tx;
using tcc::mbar_fence_init;
using tcc::mbar_init;
using tcc::smem_u32;

constexpr int kRows = 4;            // destination rows per warp
constexpr int kBatch = 8;           // neighbour rows per mbarrier phase
constexpr int kWarps = 8;
constexpr int kRowBytes = 512;
constexpr int kRingBytes = 2 * kBatch * kRowBytes;                  // per warp
constexpr int kSmemBytes = kWarps * kRingBytes + kWarps * 2 * 8;    // rings + mbarriers

// bounded wait: a wrong transaction count must not hang the device
__device__ __forceinline__ bool mbar_wait_bounded(uint32_t bar, uint32_t parity) {
  for (int it = 0; it < (1 << 22); ++it) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return true;
  }
  return false;
}

__device__ __forceinline__ void tma_row(uint32_t dst, const CUtensorMap *tm, int32_t row, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(tm), "r"(0), "r"(row), "r"(bar)
               : "memory");
}

template <int MODE>   // 0: per-row bulk copies, 1: per-row tensor-map copies
__global__ void __launch_bounds__(kWarps * 32) gather_sum_staged_kernel(const __grid_constant__ CUtensorMap tm,
                                                                        const int32_t *__restrict__ indptr,
                                                                        const int32_t *__restrict__ indices,
                                                                        const float *__restrict__ h, int32_t N,
                                                                        float *__restrict__ out, int accumulate,
                                                                        int *__restrict__ err) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t v0 = ((int64_t)blockIdx.x * kWarps + warp) * kRows;
  if (v0 >= N) return;
  const uint32_t ring = smem_u32(smem) + (uint32_t)(warp * kRingBytes);
  const uint32_t bar0 = smem_u32(smem) + (uint32_t)(kWarps * kRingBytes + warp * 16);
  if (lane == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    mbar_fence_init();
  }
  __syncwarp();
  const int nrows = (int)min((int64_t)kRows, (int64_t)N - v0);
  int32_t myptr = 0;
  if (lane <= nrows) myptr = __ldg(indptr + v0 + lane);
  const int32_t beg0 = __shfl_sync(0xffffffffu, myptr, 0);
  const int32_t total = __shfl_sync(0xffffffffu, myptr, nrows) - beg0;
  int32_t rend[kRows];
#pragma unroll
  for (int r = 0; r < kRows; ++r) rend[r] = __shfl_sync(0xffffffffu, myptr, min(r + 1, nrows)) - beg0;
  const int32_t pre = (lane < total) ? __ldg(indices + beg0 + lane) : 0;
  const int nb = (total + kBatch - 1) / kBatch;

  auto issue = [&](int b) {
    const int32_t base = b * kBatch;
    const int cnt = min(kBatch, total - base);
    const uint32_t bar = bar0 + 8u * (b & 1);
    const uint32_t dst = ring + (uint32_t)((b & 1) * kBatch * kRowBytes);
    // neighbour id of this lane's slot (lane < kBatch)
    const int32_t pos = base + lane;
    int32_t u = __shfl_sync(0xffffffffu, pre, pos & 31);
    if (pos >= 32 && lane < cnt) u = __ldg(indices + beg0 + pos);
    if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)(cnt * kRowBytes));
    __syncwarp();
    if (lane < cnt) {
      if (MODE == 0) bulk_g2s(dst + (uint32_t)(lane * kRowBytes), h + (int64_t)u * 128, kRowBytes, bar);
      else tma_row(dst + (uint32_t)(lane * kRowBytes), &tm, u, bar);
    }
  };

  float4 acc[kRows];
#pragma unroll
  for (int r = 0; r < kRows; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (nb > 0) issue(0);
  if (nb > 1) issue(1);
  bool ok = true;
  for (int b = 0; b < nb; ++b) {
    ok = mbar_wait_bounded(bar0 + 8u * (b & 1), (uint32_t)((b >> 1) & 1)) && ok;
    const float4 *slot = reinterpret_cast<const float4 *>(smem + warp * kRingBytes + (b & 1) * kBatch * kRowBytes);
    const int32_t base = b * kBatch;
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int32_t pos = base + j;
      if (pos < total) {                          // warp-uniform
        const float4 v = slot[j * 32 + lane];
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          const bool mine = (pos < rend[r]) && (r == 0 ? true : pos >= rend[r - 1]);
          if (mine) f4_add(acc[r], v);
        }
      }
    }
    if (b + 2 < nb) {
      __syncwarp();                                                    // every lane has read the buffer ...
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // ... before the async proxy overwrites it
      issue(b + 2);
    }
  }
  if (!ok && lane == 0 && err) atomicAdd(err, 1);
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    if (r < nrows) {
      float *orow = out + (v0 + r) * 128 + lane * 4;
      float4 a = acc[r];
      if (accumulate) f4_add(a, *reinterpret_cast<const float4 *>(orow));
      *reinterpret_cast<float4 *>(orow) = a;
    }
  }
}

static int *g_err_flag = nullptr;    // one int in device memory: bounded-wait failures of the last launches (development aid)

}  // namespace gtma

// cuTensorMapEncodeTiled through the runtime's driver entry point (libcuda is not linked)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int tcc::encode_f32_rows_map(const float *base, int32_t rows, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle,
                             CUtensorMap *tm) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    DDFA_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    DDFA_REQUIRE(p != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled is not available from this driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  const cuuint64_t gdim[2] = {128, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {512};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult rc = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), gdim, gstride, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DDFA_REQUIRE(rc == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)rc);
  return DDFA_OK;
}

int launch_gather_tma(int variant, const int32_t *indptr, const int32_t *indices, const float *h, int32_t N, float *out,
                      int accumulate, cudaStream_t stream) {
  using namespace gtma;
  const int64_t warps = ((int64_t)N + kRows - 1) / kRows;
  const unsigned blocks = (unsigned)((warps + kWarps - 1) / kWarps);
  if (!g_err_flag) {
    DDFA_CUDA(cudaMalloc(&g_err_flag, sizeof(int)));
    DDFA_CUDA(cudaMemset(g_err_flag, 0, sizeof(int)));
  }
  CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));
  if (variant == 10) {
    DDFA_CUDA(cudaFuncSetAttribute(gather_sum_staged_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    gather_sum_staged_kernel<0><<<blocks, kWarps * 32, kSmemBytes, stream>>>(tm, indptr, indices, h, N, out, accumulate, g_err_flag);
  } else {
    int rc = tcc::encode_f32_rows_map(h, N, 128, 1, CU_TENSOR_MAP_SWIZZLE_NONE, &tm);      // one row per copy
    if (rc) return rc;
    DDFA_CUDA(cudaFuncSetAttribute(gather_sum_staged_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    gather_sum_staged_kernel<1><<<blocks, kWarps * 32, kSmemBytes, stream>>>(tm, indptr, indices, h, N, out, accumulate, g_err_flag);
  }
  DDFA_CHECK_LAUNCH("gather_sum_staged_kernel");
  return DDFA_OK;
}

int gather_tma_errors() {
  int v = 0;
  if (gtma::g_err_flag) cudaMemcpy(&v, gtma::g_err_flag, sizeof(int), cudaMemcpyDeviceToHost);
  return v;
}

}  // namespace ddfa
