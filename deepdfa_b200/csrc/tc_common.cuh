// Shared device helpers for the tensor-core engine: mbarrier, TMA bulk copy, wgmma descriptors and instructions,
// the bf16 hi/lo operand split and the "activation image" layout.
//
// Activation image (tensor-core engine only): an [N,128] fp32 matrix X is also kept as MMA-ready operands:
//   image[tile = node/128][variant v: 0 = hi, 1 = lo][kblock kb: cols 0-63 | 64-127] = one 16 KB chunk,
//   chunk = [128 rows x 64 bf16], rows 128 B apart, 16-byte units XOR-swizzled by (row & 7)
//   (the wgmma canonical K-major SWIZZLE_128B layout; read as "MN-major" it is the [col][node] operand of the
//   weight-gradient GEMM).  hi = bf16(x), lo = bf16(x - hi).  Rows past N are zero.  64 KB per 128-node tile —
//   exactly the bytes of the fp32 matrix — so producer kernels write it instead of / next to fp32 and the GEMM
//   kernels stream it with plain 1-D TMA bulk copies (no in-kernel conversion pass).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"

namespace ddfa {
namespace tcc {

// gather_tma.cu: the tensor map of an fp32 [rows, 128] row-major plane (512-byte rows) with a box of box_cols x box_rows elements,
// encoded on the host (cuTensorMapEncodeTiled through the runtime's driver entry point).  Loads fill rows past `rows` with zeros;
// stores and reductions skip them.
int encode_f32_rows_map(const float *base, int32_t rows, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle, CUtensorMap *tm);

constexpr int kD = 128;
constexpr int kTileM = 128;
constexpr int kChunkBytes = 128 * 128;        // one [128 x 64] bf16 chunk
constexpr int kImageTileBytes = 4 * kChunkBytes;  // [hi|lo][kb0|kb1] = 64 KB per 128-node tile

__host__ __device__ __forceinline__ size_t image_bytes(int64_t n) { return (size_t)((n + kTileM - 1) / kTileM) * kImageTileBytes; }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// true in exactly one lane of a fully converged warp (lets ptxas issue the uniform-datapath tcgen05 / bulk-copy instructions
// straight-line instead of wrapping each one in a loop over "any active lane")
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xffffffff;\n"
      "@px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred));
  return pred != 0;
}
// descriptor of the same matrix `byte_off` further on in shared memory (the start-address field counts 16-byte units)
__device__ __forceinline__ uint64_t desc_advance(uint64_t desc, uint32_t byte_off) { return desc + (uint64_t)(byte_off >> 4); }

// the same with an L2 eviction-priority policy (common.cuh: l2_policy)
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar), "l"(pol)
               : "memory");
}

// ---- warpgroup MMA (sm_90a wgmma) ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor: start >> 4 in bits 0-13, leading byte offset >> 4 in 16-29, stride byte offset >> 4 in 32-45,
// layout in 62-63 (1 = SWIZZLE_128B).  Every operand here is a stack of 128-byte rows in 1024-byte groups of eight (SBO = 1024).
//   K-major (A or B, no transpose): rows = M or N, 64 bf16 of K per row; LBO is unused for swizzled K-major layouts.  A K step of
//     16 advances the start address by 32 bytes inside the swizzle atom.
//   MN-major (transposed): rows = K, 64 consecutive M / N elements per row; LBO = byte distance to the next 64 M / N elements.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes = 16u) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma_wait()
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Accumulator fragment of an m64nN wgmma: thread t of the warpgroup holds element d[4 j + 2 h + e] =
// D[16 (t / 32) + (t % 32) / 4 + 8 h][8 j + 2 (t % 4) + e]   (h, e in {0, 1}, j < N / 8).

// D[64 x 64] (+)= A[64 x 16] * B[16 x 64], bf16 operands from shared memory, fp32 accumulator in registers
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
}

// D[64 x 96] (+)= A[64 x 16] * B[16 x 96], bf16 operands from shared memory, fp32 accumulator in registers
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n96(float (&d)[48], uint64_t a, uint64_t b, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, %51, %52;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
}

// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], bf16 operands from shared memory, fp32 accumulator in registers
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
}

// wait bounded in time: a protocol error ends the kernel with a trap instead of hanging the device
__device__ __forceinline__ void mbar_wait_bounded(uint32_t bar, uint32_t parity) {
  for (uint32_t it = 0; it < (1u << 24); ++it) {
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
    if (done) return;
  }
  __trap();
}


// byte offset of element (row, k) inside a [rows x 64] bf16 K-major SWIZZLE_128B chunk
__host__ __device__ __forceinline__ uint32_t sw128_offset(int row, int k) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + (k & 7) * 2);
}
// byte offset of element (node, col) variant v inside an activation image
__host__ __device__ __forceinline__ size_t image_offset(int64_t node, int col, int v) {
  return (size_t)(node / kTileM) * kImageTileBytes + (size_t)((v * 2 + (col >> 6)) * kChunkBytes) +
         sw128_offset((int)(node % kTileM), col & 63);
}
// The same layout for a matrix of D columns (D a multiple of 64): a 128-row tile is [hi | lo][D / 64 column chunks] of 16 KB,
// 128 x D x 4 bytes.  D = 128 is the activation image above.  The wide-width engine (gru_tc_wide.cu) keeps every GEMM operand so.
__host__ __device__ __forceinline__ size_t image_bytes_w(int64_t n, int D) { return (size_t)((n + kTileM - 1) / kTileM) * kTileM * 4 * (size_t)D; }
__host__ __device__ __forceinline__ size_t image_offset_w(int64_t node, int col, int v, int D) {
  return (size_t)(node / kTileM) * ((size_t)kTileM * 4 * D) + (size_t)((v * (D >> 6) + (col >> 6)) * kChunkBytes) +
         sw128_offset((int)(node % kTileM), col & 63);
}

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16 &hi, __nv_bfloat16 &lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// 4 consecutive fp32 -> packed 4 x bf16 hi and 4 x bf16 lo (8 bytes each).  Two values per conversion instruction
// (cvt.rn.bf16x2.f32 = F2FP.BF16.F32.PACK_AB, which also does the packing) instead of eight scalar F2F on the quarter-rate
// conversion pipe plus shifts and ORs; the values are those of split_bf16 (both round to nearest even).
__device__ __forceinline__ uint32_t bf16x2_bits(float lo_half, float hi_half) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo_half, hi_half);      // .x -> bits 0-15, .y -> bits 16-31
  return *reinterpret_cast<const uint32_t *>(&v);
}
__device__ __forceinline__ void split4(const float4 &x, uint2 &ph, uint2 &pl) {
  ph.x = bf16x2_bits(x.x, x.y);
  ph.y = bf16x2_bits(x.z, x.w);
  pl.x = bf16x2_bits(x.x - __uint_as_float(ph.x << 16), x.y - __uint_as_float(ph.x & 0xffff0000u));
  pl.y = bf16x2_bits(x.z - __uint_as_float(ph.y << 16), x.w - __uint_as_float(ph.y & 0xffff0000u));
}
// 8 consecutive fp32 (one 16-byte bf16 unit) -> hi / lo uint4
__device__ __forceinline__ void split8(const float (&x)[8], uint4 &ph, uint4 &pl) {
  uint2 h0, l0, h1, l1;
  split4(make_float4(x[0], x[1], x[2], x[3]), h0, l0);
  split4(make_float4(x[4], x[5], x[6], x[7]), h1, l1);
  ph = make_uint4(h0.x, h0.y, h1.x, h1.y);
  pl = make_uint4(l0.x, l0.y, l1.x, l1.y);
}

// ---- saved gate values of one element, 64 bits: r, z in [0,1] as 14-bit fixed point, n in [-1,1] as 16-bit fixed point, gh_n as a
// 20-bit float (1 sign, 5 exponent bits with fp16's bias, 14 mantissa bits).  Absolute error <= 3.1e-5 on r, z, 1.6e-5 on n, relative
// 3.1e-5 on gh_n (|gh_n| < 6.1e-5 flushes to 0) — an order below plain fp16 (2.4e-4 / 4.9e-4), which measurably moved the parameter
// gradients (profiles/r03b: 1.6e-5 -> 2e-4 relative), at the same 8 bytes.  Layout: x = r | z << 14 | gh[3:0] << 28 ; y = n | gh[19:4] << 16.
// gh_n = +-inf and a NaN anywhere in the element are kept (exponent code 31), so the gate backward sees them as torch's does.
__device__ __forceinline__ uint2 pack_gates(float r, float z, float n, float ghn) {
  // r, z come out of fast_sigmoid (in [0,1]) and n out of fast_tanh (in [-1,1]): no clamping needed.  Rounding to the nearest
  // integer by adding 2^23 (1.5 * 2^23 for the signed value) inside an FMA and reading the low mantissa bits: one FFMA on the
  // main pipe instead of FMUL + F2I (the forward epilogue's conversion / MUFU pipe is its busiest unit), and a single rounding.
  const uint32_t rq = __float_as_uint(fmaf(r, 16383.f, 8388608.f)) & 0x3fffu, zq = __float_as_uint(fmaf(z, 16383.f, 8388608.f)) & 0x3fffu;
  const uint32_t nq = __float_as_uint(fmaf(n, 32767.f, 12582912.f)) & 0xffffu;
  const uint32_t b = __float_as_uint(ghn);
  // round the mantissa to 14 bits (a carry runs into the exponent, as it should), drop the sign, re-bias the exponent 127 -> 15:
  // core = [exponent - 112 | mantissa] ; below 2^-14 -> 0, a finite value above fp16's range -> the largest finite code
  const int core = (int)(((b + 0x100u) << 1) >> 10) - (112 << 14);
  uint32_t g = core < (1 << 14) ? 0u : (uint32_t)min(core, (31 << 14) - 1);
  // Non-finite values take fp16's codes, exponent 31, which no finite value reaches: gh_n = +-inf keeps its sign with a zero
  // mantissa; a NaN in r, z, n or gh_n makes the whole element NaN (mantissa 1), as every gate gradient of that element is NaN in
  // torch then.  r, z and n are bounded, so their sum with gh_n is non-finite exactly when one of these holds.
  const float t = r + z + n + ghn;
  if (!(fabsf(t) < INFINITY)) g = (31u << 14) | (t != t ? 1u : 0u);
  g |= (b >> 12) & 0x80000u;
  return make_uint2(rq | (zq << 14) | (g << 28), nq | ((g >> 4) << 16));
}
__device__ __forceinline__ void unpack_gates(const uint2 &p, float &r, float &z, float &n, float &ghn) {
  r = (float)(p.x & 0x3fffu) * (1.f / 16383.f);
  z = (float)((p.x >> 14) & 0x3fffu) * (1.f / 16383.f);
  // signed 16-bit -> float without I2F: (value + 32768) placed in the mantissa of 2^23, minus (2^23 + 32768) — exact
  n = (__uint_as_float(((p.y & 0xffffu) ^ 0x4b008000u)) - 8421376.f) * (1.f / 32767.f);
  const uint32_t g = ((p.y >> 16) << 4) | (p.x >> 28);
  const uint32_t e = (g >> 14) & 31u;
  ghn = e == 0u ? 0.f : __uint_as_float(((g >> 19) << 31) | ((e == 31u ? 255u : e + 112u) << 23) | ((g & 0x3fffu) << 9));
  if (ghn != ghn) r = z = n = ghn;      // pack_gates' NaN code: the element's gates were not finite
}

// Gate math on the MUFU pipe.  __expf() expands to ex2.approx WITHOUT .ftz plus a range fix-up (FSETP, two predicated FMULs) per
// call — three calls per output element in the forward epilogue, which is bound by its instruction count; flushing the (here
// irrelevant) denormal results instead saves 9 instructions per element.  ex2.approx.ftz: 2^-22 relative; rcp.approx.ftz: 1 ulp.
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_sigmoid(float x) { return rcp_ftz(1.f + ex2_ftz(-1.4426950408889634f * x)); }
__device__ __forceinline__ float fast_tanh(float x) {
  const float e = ex2_ftz(2.885390081777927f * x);  // e^(2x): inf for large x -> 1 - 0 = 1 ; 0 for very negative x -> 1 - 2 = -1
  return fmaf(-2.f, rcp_ftz(e + 1.f), 1.f);
}

// ---- pipeline timeline (development aid; ddfa_debug_set key 2 switches it on, ddfa_debug_read fetches it) -----------
// Each translation unit that includes this header gets its own buffer: [CTA][tile][event] SM-clock stamps.
constexpr int kTraceCtas = 132, kTraceTiles = 12, kTraceEvents = 16;
constexpr size_t kTraceWords = (size_t)kTraceCtas * kTraceTiles * kTraceEvents;
static __device__ long long g_trace[kTraceWords];
static __device__ int g_trace_on = 0;
__device__ __forceinline__ void trace_put(int on, int tile_i, int ev, long long v) {
  if (on && blockIdx.x < kTraceCtas && tile_i < kTraceTiles) g_trace[((size_t)blockIdx.x * kTraceTiles + tile_i) * kTraceEvents + ev] = v;
}
__device__ __forceinline__ void trace_stamp(int on, int tile_i, int ev) { trace_put(on, tile_i, ev, clock64()); }

}  // namespace tcc
}  // namespace ddfa
