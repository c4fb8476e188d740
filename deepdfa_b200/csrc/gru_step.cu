// K4 — one GRU propagation step (torch.nn.GRUCell inside DGL GatedGraphConv, reference call site
// DDFA/code_gnn/models/flow_gnn/ggnn.py:95; gate order r,z,n) and its backward.
//
// Uses the folded formulation (SURVEY.md App. A): with s = A h (raw gather-sum, K3)
//     gi = s w_fold^T + indeg * b_fold + b_ih        w_fold = W_ih W, b_fold = W_ih b
//     gh = h w_hh^T + b_hh
// which equals GRUCell(a, h) for a_v = sum_{u->v} (W h_u + b).
//
// This file holds the engine dispatch, the SIMT engine (fp32 FFMA GEMMs from sgemm.cu + fused
// gate kernels) and the weight-folding helpers.  The tcgen05 engine lives in gru_tc_fwd3.cu / gru_tc_bwd.cu (D == 128) and
// gru_tc_wide.cu (D = 192 .. 512, D % 64 == 0: the SIMT data flow below with tensor-core GEMMs in place of the sgemm calls).
#include "common.cuh"

namespace ddfa {

// ---- gate math, forward ------------------------------------------------------------------
// gi_raw/gh_raw: [N,3D] GEMM outputs without biases.  gates: [4][N][D] = r, z, n, gh_n (+b_hh_n).
__global__ void __launch_bounds__(256) gru_gate_fwd_kernel(const float *__restrict__ gi_raw, const float *__restrict__ gh_raw,
                                                           const float *__restrict__ h, const int32_t *__restrict__ indptr,
                                                           const float *__restrict__ b_fold, const float *__restrict__ b_ih,
                                                           const float *__restrict__ b_hh, int32_t N, int32_t D,
                                                           float *__restrict__ h_out, float *__restrict__ gates) {
  const int dq = D >> 2;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (int64_t)N * dq) return;
  const int32_t n = (int32_t)(t / dq);
  const int c = (int)(t - (int64_t)n * dq) * 4;
  const float deg = (float)(indptr[n + 1] - indptr[n]);
  const float *gi = gi_raw + (int64_t)n * 3 * D;
  const float *gh = gh_raw + (int64_t)n * 3 * D;
  const float4 hv = *reinterpret_cast<const float4 *>(h + (int64_t)n * D + c);
  float4 g[3][2];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const float4 a = *reinterpret_cast<const float4 *>(gi + q * D + c);
    const float4 bf = *reinterpret_cast<const float4 *>(b_fold + q * D + c);
    const float4 bi = *reinterpret_cast<const float4 *>(b_ih + q * D + c);
    g[q][0] = make_float4(fmaf(deg, bf.x, a.x) + bi.x, fmaf(deg, bf.y, a.y) + bi.y, fmaf(deg, bf.z, a.z) + bi.z,
                          fmaf(deg, bf.w, a.w) + bi.w);
    const float4 b = *reinterpret_cast<const float4 *>(gh + q * D + c);
    const float4 bh = *reinterpret_cast<const float4 *>(b_hh + q * D + c);
    g[q][1] = make_float4(b.x + bh.x, b.y + bh.y, b.z + bh.z, b.w + bh.w);
  }
  float4 r, z, nn, o;
#define GATE(f)                                            \
  r.f = sigmoidf_acc(g[0][0].f + g[0][1].f);               \
  z.f = sigmoidf_acc(g[1][0].f + g[1][1].f);               \
  nn.f = tanhf(fmaf(r.f, g[2][1].f, g[2][0].f));           \
  o.f = fmaf(z.f, hv.f - nn.f, nn.f);
  GATE(x) GATE(y) GATE(z) GATE(w)
#undef GATE
  *reinterpret_cast<float4 *>(h_out + (int64_t)n * D + c) = o;
  if (gates) {
    const int64_t plane = (int64_t)N * D, off = (int64_t)n * D + c;
    *reinterpret_cast<float4 *>(gates + off) = r;
    *reinterpret_cast<float4 *>(gates + plane + off) = z;
    *reinterpret_cast<float4 *>(gates + 2 * plane + off) = nn;
    *reinterpret_cast<float4 *>(gates + 3 * plane + off) = g[2][1];
  }
}

// ---- gate math, backward -----------------------------------------------------------------
// dgi, dgh: [N,3D] (inputs of the dgrad/wgrad GEMMs).  dh_part = dh_out * z.
// Bias grads accumulated with one RED per column per CTA, or (bias_slots != NULL, deterministic mode) written to the CTA's slot
// [7][D] and added in CTA order by bias_slots_sum_kernel.
constexpr int kGateBwdRows = 128;
__global__ void __launch_bounds__(256) gru_gate_bwd_kernel(const float *__restrict__ dh_out, const float *__restrict__ h,
                                                           const float *__restrict__ gates, const int32_t *__restrict__ indptr,
                                                           int32_t N, int32_t D, float *__restrict__ dgi, float *__restrict__ dgh,
                                                           float *__restrict__ dh_part, float *__restrict__ db_fold,
                                                           float *__restrict__ db_ih, float *__restrict__ db_hh,
                                                           float *__restrict__ bias_slots) {
  extern __shared__ float red[];  // [blockDim.y][7][D]
  const int c = threadIdx.x * 4;
  const int64_t plane = (int64_t)N * D;
  float4 acc[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int32_t row0 = blockIdx.x * kGateBwdRows;
  const int32_t row1 = min(N, row0 + kGateBwdRows);
  for (int32_t n = row0 + threadIdx.y; n < row1; n += blockDim.y) {
    const int64_t off = (int64_t)n * D + c;
    const float deg = (float)(indptr[n + 1] - indptr[n]);
    const float4 d = *reinterpret_cast<const float4 *>(dh_out + off);
    const float4 hv = *reinterpret_cast<const float4 *>(h + off);
    const float4 r = *reinterpret_cast<const float4 *>(gates + off);
    const float4 z = *reinterpret_cast<const float4 *>(gates + plane + off);
    const float4 nn = *reinterpret_cast<const float4 *>(gates + 2 * plane + off);
    const float4 ghn = *reinterpret_cast<const float4 *>(gates + 3 * plane + off);
    float4 qr, qz, qn, qnr, dhp;
#define BWD(f)                                               \
  {                                                          \
    const float dz = d.f * (hv.f - nn.f);                    \
    const float dn = d.f * (1.f - z.f);                      \
    dhp.f = d.f * z.f;                                       \
    qn.f = dn * (1.f - nn.f * nn.f);                         \
    qz.f = dz * z.f * (1.f - z.f);                           \
    qr.f = qn.f * ghn.f * r.f * (1.f - r.f);                 \
    qnr.f = qn.f * r.f;                                      \
  }
    BWD(x) BWD(y) BWD(z) BWD(w)
#undef BWD
    float *gi = dgi + (int64_t)n * 3 * D + c;
    float *gh = dgh + (int64_t)n * 3 * D + c;
    *reinterpret_cast<float4 *>(gi) = qr;
    *reinterpret_cast<float4 *>(gi + D) = qz;
    *reinterpret_cast<float4 *>(gi + 2 * D) = qn;
    *reinterpret_cast<float4 *>(gh) = qr;
    *reinterpret_cast<float4 *>(gh + D) = qz;
    *reinterpret_cast<float4 *>(gh + 2 * D) = qnr;
    *reinterpret_cast<float4 *>(dh_part + off) = dhp;
    f4_add(acc[0], qr); f4_add(acc[1], qz); f4_add(acc[2], qn); f4_add(acc[3], qnr);
    f4_fma(acc[4], deg, qr); f4_fma(acc[5], deg, qz); f4_fma(acc[6], deg, qn);
  }
  // reduce over threadIdx.y
#pragma unroll
  for (int i = 0; i < 7; ++i) *reinterpret_cast<float4 *>(&red[((int64_t)threadIdx.y * 7 + i) * D + c]) = acc[i];
  __syncthreads();
  if (threadIdx.y == 0) {
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      float4 sum = acc[i];
      for (int y = 1; y < blockDim.y; ++y) f4_add(sum, *reinterpret_cast<const float4 *>(&red[((int64_t)y * 7 + i) * D + c]));
      acc[i] = sum;
    }
    if (bias_slots) {
#pragma unroll
      for (int i = 0; i < 7; ++i) *reinterpret_cast<float4 *>(bias_slots + ((int64_t)blockIdx.x * 7 + i) * D + c) = acc[i];
      return;
    }
#define RED4(ptr, v) atomicAdd((ptr) + 0, (v).x); atomicAdd((ptr) + 1, (v).y); atomicAdd((ptr) + 2, (v).z); atomicAdd((ptr) + 3, (v).w);
    RED4(db_ih + c, acc[0]) RED4(db_ih + D + c, acc[1]) RED4(db_ih + 2 * D + c, acc[2])
    RED4(db_hh + c, acc[0]) RED4(db_hh + D + c, acc[1]) RED4(db_hh + 2 * D + c, acc[3])
    RED4(db_fold + c, acc[4]) RED4(db_fold + D + c, acc[5]) RED4(db_fold + 2 * D + c, acc[6])
#undef RED4
  }
}

// one thread per bias-gradient element (7 x D): the CTAs' slots added in CTA order, then into db_ih / db_hh / db_fold as above
__global__ void __launch_bounds__(256) bias_slots_sum_kernel(const float *__restrict__ slots, int ctas, int32_t D, float *__restrict__ db_fold,
                                                             float *__restrict__ db_ih, float *__restrict__ db_hh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 7 * D) return;
  float v = 0.f;
  for (int c = 0; c < ctas; ++c) v += slots[(int64_t)c * 7 * D + i];
  const int which = i / D, col = i - which * D;
  if (which < 3) db_ih[which * D + col] += v;
  if (which < 2) db_hh[which * D + col] += v;
  if (which == 3) db_hh[2 * D + col] += v;
  if (which >= 4) db_fold[(which - 4) * D + col] += v;
}

// split of the SIMT weight-gradient GEMMs (K = N nodes) over the SMs
static int simt_wgrad_split(int32_t N, int32_t D) {
  const int tiles = ((3 * D + 127) / 128) * ((D + 127) / 128);
  int split = (2 * kNumSMs + tiles - 1) / tiles;
  const int k_tiles = (N + 15) / 16;
  if (split > k_tiles / 8) split = k_tiles / 8 > 0 ? k_tiles / 8 : 1;
  return split;
}

// ---- fold helpers --------------------------------------------------------------------------
// b_fold[j] = sum_k w_ih[j,k] b[k]   (3D rows, warp per row)
__global__ void fold_bias_kernel(const float *__restrict__ w_ih, const float *__restrict__ b, int32_t D, float *__restrict__ b_fold) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= 3 * D) return;
  float s = 0.f;
  for (int k = lane; k < D; k += 32) s = fmaf(w_ih[(int64_t)row * D + k], b[k], s);
  s = warp_sum(s);
  if (lane == 0) b_fold[row] = s;
}
// dw_ih[j,k] += db_fold[j] * b[k]
__global__ void fold_bias_bwd_outer_kernel(const float *__restrict__ db_fold, const float *__restrict__ b, int32_t D, float *__restrict__ dw_ih) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (int64_t)3 * D * D) return;
  const int j = (int)(t / D), k = (int)(t % D);
  dw_ih[t] = fmaf(db_fold[j], b[k], dw_ih[t]);
}
// db[k] += sum_j w_ih[j,k] db_fold[j]     block = (32 columns) x (8 row partitions), coalesced along k
__global__ void __launch_bounds__(256) fold_bias_bwd_vec_kernel(const float *__restrict__ w_ih, const float *__restrict__ db_fold,
                                                                int32_t D, float *__restrict__ db) {
  __shared__ float red[8][33];
  const int k = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (k < D)
    for (int j = threadIdx.y; j < 3 * D; j += 8) s = fmaf(w_ih[(int64_t)j * D + k], db_fold[j], s);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && k < D) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += red[y][threadIdx.x];
    db[k] += t;
  }
}

}  // namespace ddfa

extern "C" {

int ddfa_fold_weights_fwd(const float *w_msg, const float *b_msg, const float *w_ih, int32_t D, float *w_fold,
                          float *b_fold, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(D > 0 && D % 4 == 0, "ddfa_fold_weights_fwd: D=%d must be a positive multiple of 4", D);
  DDFA_REQUIRE(w_msg && b_msg && w_ih && w_fold && b_fold, "ddfa_fold_weights_fwd: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  // w_fold[3D,D] = w_ih[3D,D] @ w_msg[D,D]
  int rc = sgemm(0, 0, 3 * D, D, D, 1.f, w_ih, D, w_msg, D, 0.f, w_fold, D, 1, stream);
  if (rc) return rc;
  fold_bias_kernel<<<(3 * D + 7) / 8, 256, 0, stream>>>(w_ih, b_msg, D, b_fold);
  DDFA_CHECK_LAUNCH("fold_bias_kernel");
  return DDFA_OK;
}

int ddfa_fold_weights_bwd(const float *w_msg, const float *b_msg, const float *w_ih, const float *dw_fold,
                          const float *db_fold, int32_t D, float *dw_msg, float *db_msg, float *dw_ih, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(D > 0 && D % 4 == 0, "ddfa_fold_weights_bwd: D=%d must be a positive multiple of 4", D);
  DDFA_REQUIRE(w_msg && b_msg && w_ih && dw_fold && db_fold && dw_msg && db_msg && dw_ih, "ddfa_fold_weights_bwd: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  // dW_ih += dw_fold @ W^T
  int rc = sgemm(0, 1, 3 * D, D, D, 1.f, dw_fold, D, w_msg, D, 1.f, dw_ih, D, 1, stream);
  if (rc) return rc;
  // dW += W_ih^T @ dw_fold
  rc = sgemm(1, 0, D, D, 3 * D, 1.f, w_ih, D, dw_fold, D, 1.f, dw_msg, D, 1, stream);
  if (rc) return rc;
  const int64_t tot = (int64_t)3 * D * D;
  fold_bias_bwd_outer_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(db_fold, b_msg, D, dw_ih);
  DDFA_CHECK_LAUNCH("fold_bias_bwd_outer_kernel");
  fold_bias_bwd_vec_kernel<<<(D + 31) / 32, dim3(32, 8), 0, stream>>>(w_ih, db_fold, D, db_msg);
  DDFA_CHECK_LAUNCH("fold_bias_bwd_vec_kernel");
  return DDFA_OK;
}

size_t ddfa_gru_step_workspace_bytes(int32_t N, int32_t D, int engine) {
  if (N < 0 || D <= 0) return 0;
  // tcgen05: [packed per-slice weight images + biases][s image][h image]; the two images are only used by the
  // fp32-in/fp32-out entry ddfa_gru_step_fwd (N = 0 gives the size ddfa_gru_step_fwd_image needs).
  if (engine == DDFA_ENGINE_TCGEN05 && D == 128) return ddfa::gru_tc2_workspace_bytes() + 2 * ddfa::act_image_bytes(N);
  if (engine == DDFA_ENGINE_TCGEN05 && !ddfa::gru_tcw_width(D)) return 16;
  // tcgen05 at the wide widths: [W' and Whh operand images (ddfa_gru_step_prepare)][gi|gh][s and h images]
  const size_t planes = sizeof(float) * 2 * (size_t)N * 3 * (size_t)D;  // gi|gh
  if (engine == DDFA_ENGINE_TCGEN05) return ddfa::gru_tcw_weights_bytes(D) + planes + ddfa::gru_tcw_fwd_scratch_bytes(N, D);
  return planes;
}

size_t ddfa_act_image_bytes(int64_t num_nodes) { return num_nodes < 0 ? 0 : ddfa::act_image_bytes(num_nodes); }

int ddfa_act_to_image(const float *x, int32_t N, int32_t D, void *image, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_act_to_image: activation images exist for D == 128 only (N=%d D=%d)", N, D);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(x && image && aligned16(x) && aligned16(image), "ddfa_act_to_image: NULL or unaligned pointer");
  return act_to_image(x, N, image, as_stream(stream_));
}

int ddfa_gru_step_fwd_image(const void *s_image, const void *h_image, const float *h, const int32_t *indptr, int32_t N,
                            int32_t D, float *h_out, void *h_out_image, float *save_gates, const void *workspace,
                            size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gru_step_fwd_image: the tcgen05 engine supports D == 128 only (N=%d D=%d)", N, D);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(s_image && h_image && h && indptr && h_out, "ddfa_gru_step_fwd_image: NULL pointer");
  return gru_tc2_step_fwd(s_image, h_image, h, indptr, N, h_out, h_out_image, save_gates, nullptr, workspace, workspace_bytes,
                          as_stream(stream_));
}

size_t ddfa_gru_gates_packed_bytes(int32_t N, int32_t D) { return (N < 0 || D <= 0) ? 0 : (size_t)N * (size_t)D * 8; }

int ddfa_gru_step_fwd_image_v2(const void *s_image, const void *h_image, const float *h, const int32_t *indptr, int32_t N, int32_t D,
                               float *h_out, void *h_out_image, void *save_gates_packed, const void *workspace, size_t workspace_bytes,
                               void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gru_step_fwd_image_v2: the tcgen05 engine supports D == 128 only (N=%d D=%d)", N, D);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(s_image && h_image && indptr, "ddfa_gru_step_fwd_image_v2: NULL pointer");
  DDFA_REQUIRE(h_out || h_out_image, "ddfa_gru_step_fwd_image_v2: neither h_out nor h_out_image given");
  return gru_tc2_step_fwd(s_image, h_image, h, indptr, N, h_out, h_out_image, nullptr, save_gates_packed, workspace, workspace_bytes,
                          as_stream(stream_));
}

static int check_step_args(const char *who, int32_t N, int32_t D, int engine) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D > 0 && D % 4 == 0 && D <= 1024, "%s: unsupported shape N=%d D=%d", who, N, D);
  DDFA_REQUIRE(engine == DDFA_ENGINE_SIMT || engine == DDFA_ENGINE_TCGEN05, "%s: unknown engine %d", who, engine);
  if (engine == DDFA_ENGINE_TCGEN05 && D != 128 && !gru_tcw_width(D)) {
    set_error("%s: the tcgen05 engine supports D = 128, 192, 256, 320, 384, 448 and 512 only (got %d); select DDFA_ENGINE_SIMT", who, D);
    return DDFA_ERR_UNSUPPORTED;
  }
  return DDFA_OK;
}

int ddfa_gru_step_prepare(const float *w_fold, const float *b_fold, const float *b_ih, const float *w_hh, const float *b_hh,
                          int32_t D, int engine, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  int rc = check_step_args("ddfa_gru_step_prepare", 0, D, engine);
  if (rc) return rc;
  if (engine == DDFA_ENGINE_SIMT) return DDFA_OK;  // nothing to pre-pack
  DDFA_REQUIRE(w_fold && b_fold && b_ih && w_hh && b_hh, "ddfa_gru_step_prepare: NULL pointer");
  if (D != 128) {      // the W' and Whh operand images at the head of the workspace
    if (workspace == nullptr || workspace_bytes < gru_tcw_weights_bytes(D)) {
      set_error("ddfa_gru_step_prepare: workspace too small (%zu < %zu)", workspace_bytes, gru_tcw_weights_bytes(D));
      return DDFA_ERR_WORKSPACE;
    }
    DDFA_REQUIRE(aligned16(w_fold) && aligned16(w_hh), "ddfa_gru_step_prepare: w_fold / w_hh not 16-byte aligned");
    return gru_tcw_prepare(w_fold, w_hh, D, workspace, as_stream(stream_));
  }
  return gru_tc2_prepare(w_fold, b_fold, b_ih, w_hh, b_hh, workspace, workspace_bytes, as_stream(stream_));
}

int ddfa_gru_step_fwd(const float *s, const float *h, const int32_t *indptr, const float *w_fold, const float *b_fold,
                      const float *b_ih, const float *w_hh, const float *b_hh, int32_t N, int32_t D, float *h_out,
                      float *save_gates, void *workspace, size_t workspace_bytes, int engine, void *stream_) {
  using namespace ddfa;
  int rc = check_step_args("ddfa_gru_step_fwd", N, D, engine);
  if (rc) return rc;
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(s && h && indptr && w_fold && b_fold && b_ih && w_hh && b_hh && h_out, "ddfa_gru_step_fwd: NULL pointer");
  cudaStream_t stream = as_stream(stream_);
  if (workspace_bytes < ddfa_gru_step_workspace_bytes(N, D, engine) || workspace == nullptr) {
    set_error("ddfa_gru_step_fwd: workspace too small (%zu < %zu)", workspace_bytes, ddfa_gru_step_workspace_bytes(N, D, engine));
    return DDFA_ERR_WORKSPACE;
  }
  if (engine == DDFA_ENGINE_TCGEN05 && D == 128) {
    // fp32-in / fp32-out convenience path (tests, tools): build the two operand images in the workspace, then run the
    // image kernel.  The training driver calls ddfa_gru_step_fwd_image with images written by the producer kernels.
    uint8_t *ws8 = static_cast<uint8_t *>(workspace);
    void *s_img = ws8 + gru_tc2_workspace_bytes();
    void *h_img = ws8 + gru_tc2_workspace_bytes() + act_image_bytes(N);
    rc = act_to_image(s, N, s_img, stream);
    if (rc) return rc;
    rc = act_to_image(h, N, h_img, stream);
    if (rc) return rc;
    return gru_tc2_step_fwd(s_img, h_img, h, indptr, N, h_out, nullptr, save_gates, nullptr, workspace, workspace_bytes, stream);
  }
  const bool wide = engine == DDFA_ENGINE_TCGEN05;       // D = 192 .. 512: tensor-core GEMMs, the rest as SIMT
  const size_t head = wide ? gru_tcw_weights_bytes(D) : 0;
  float *gi = reinterpret_cast<float *>(static_cast<uint8_t *>(workspace) + head);
  float *gh = gi + (size_t)N * 3 * D;
  if (wide) {
    // s and h become operand images through 16-byte loads
    DDFA_REQUIRE(aligned16(s) && aligned16(h), "ddfa_gru_step_fwd: s / h not 16-byte aligned");
    rc = gru_tcw_fwd_gemms(s, h, N, D, workspace, gh + (size_t)N * 3 * D, gi, gh, stream);
  } else {
    rc = sgemm(0, 1, N, 3 * D, D, 1.f, s, D, w_fold, D, 0.f, gi, 3 * D, 1, stream);
    if (rc) return rc;
    rc = sgemm(0, 1, N, 3 * D, D, 1.f, h, D, w_hh, D, 0.f, gh, 3 * D, 1, stream);
  }
  if (rc) return rc;
  const int64_t tot = (int64_t)N * (D / 4);
  gru_gate_fwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(gi, gh, h, indptr, b_fold, b_ih, b_hh, N, D, h_out, save_gates);
  DDFA_CHECK_LAUNCH("gru_gate_fwd_kernel");
  return DDFA_OK;
}

size_t ddfa_gru_step_bwd_workspace_bytes(int32_t N, int32_t D, int engine) {
  if (N < 0 || D <= 0) return 0;
  return ddfa_gru_step_bwd_workspace_bytes_steps(N, D, engine, 1);
}

size_t ddfa_gru_step_bwd_workspace_bytes_steps(int32_t N, int32_t D, int engine, int32_t steps) {
  if (N < 0 || D <= 0) return 0;
  if (engine == DDFA_ENGINE_TCGEN05 && D == 128) return ddfa::gru_tc2_bwd_workspace_bytes(N, steps);   // layout: gru_tc_bwd.cu
  if (engine == DDFA_ENGINE_TCGEN05 && !ddfa::gru_tcw_width(D)) return 16;
  // dgi | dgh | bias slots of the gate-backward CTAs | split-K slices of one weight gradient (the last two: deterministic mode,
  // reserved in both modes).  tcgen05 at the wide widths: [W' and Whh operand images] dgi | dgh | bias slots [operand images
  // and weight-gradient slices: gru_tc_wide.cu] (the step count does not matter: the weight gradient is taken per step)
  const size_t slots = (size_t)((N + ddfa::kGateBwdRows - 1) / ddfa::kGateBwdRows) * 7 * D;
  const size_t planes = sizeof(float) * (2 * (size_t)N * 3 * (size_t)D + slots);
  if (engine == DDFA_ENGINE_TCGEN05) return ddfa::gru_tcw_weights_bytes(D) + planes + ddfa::gru_tcw_bwd_scratch_bytes(N, D);
  const size_t part = (size_t)ddfa::sgemm_splitk_ordered_slices(N, ddfa::simt_wgrad_split(N, D)) * 3 * D * D;
  return planes + sizeof(float) * part;
}

int ddfa_gru_bwd_wgrad_batched(const void *const *s_images, const void *const *h_images, int32_t steps, int32_t N, int32_t D,
                               float *dw_fold, float *dw_hh, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gru_bwd_wgrad_batched: the tcgen05 engine supports D == 128 only (N=%d D=%d)", N, D);
  DDFA_REQUIRE(s_images && h_images && dw_fold && dw_hh, "ddfa_gru_bwd_wgrad_batched: NULL pointer");
  if (N == 0) return DDFA_OK;
  return gru_tc2_bwd_wgrad_batched(s_images, h_images, steps, N, dw_fold, dw_hh, workspace, workspace_bytes, as_stream(stream_));
}

int ddfa_gru_step_bwd_image(const float *dh_out, const float *ds_prev, const int32_t *indptr_t, const int32_t *indices_t,
                            const float *h, const void *h_image, const void *s_image, const float *gates,
                            const int32_t *indptr, int32_t N, int32_t D, float *ds, float *dh, float *dw_fold, float *db_fold,
                            float *db_ih, float *dw_hh, float *db_hh, void *workspace, size_t workspace_bytes, int wgrad_mode,
                            void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gru_step_bwd_image: the tcgen05 engine supports D == 128 only (N=%d D=%d)", N, D);
  DDFA_REQUIRE((wgrad_mode >= 0 && wgrad_mode <= 2) || (wgrad_mode >= 16 && wgrad_mode < 32),
               "ddfa_gru_step_bwd_image: wgrad_mode must be 0, 1, 2 or DDFA_WGRAD_KEEP(slot < 16) (got %d)", wgrad_mode);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(dh_out && h && s_image && gates && indptr && ds && dh && dw_fold && db_fold && db_ih && dw_hh && db_hh,
               "ddfa_gru_step_bwd_image: NULL pointer");
  DDFA_REQUIRE(dh != dh_out, "ddfa_gru_step_bwd_image: dh must not alias dh_out");
  DDFA_REQUIRE(ds_prev == nullptr || (indptr_t && indices_t), "ddfa_gru_step_bwd_image: ds_prev given without the transposed CSR");
  DDFA_REQUIRE(ds_prev == nullptr || ds_prev != ds, "ddfa_gru_step_bwd_image: ds must not alias ds_prev");
  return gru_tc2_step_bwd(dh_out, ds_prev, indptr_t, indices_t, h, h_image, s_image, gates, nullptr, indptr, N, ds, dh, dw_fold, db_fold, db_ih, dw_hh, db_hh, workspace,
                          workspace_bytes, wgrad_mode, as_stream(stream_));
}

int ddfa_gru_step_bwd_image_v2(const float *dh_out, const float *ds_prev, const int32_t *indptr_t, const int32_t *indices_t,
                               const float *h, const void *h_image, const void *s_image, const void *gates_packed,
                               const int32_t *indptr, int32_t N, int32_t D, float *ds, float *dh, float *dw_fold, float *db_fold,
                               float *db_ih, float *dw_hh, float *db_hh, void *workspace, size_t workspace_bytes, int wgrad_mode,
                               void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128, "ddfa_gru_step_bwd_image_v2: the tcgen05 engine supports D == 128 only (N=%d D=%d)", N, D);
  DDFA_REQUIRE((wgrad_mode >= 0 && wgrad_mode <= 2) || (wgrad_mode >= 16 && wgrad_mode < 32),
               "ddfa_gru_step_bwd_image_v2: wgrad_mode must be 0, 1, 2 or DDFA_WGRAD_KEEP(slot < 16) (got %d)", wgrad_mode);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(dh_out && h_image && s_image && gates_packed && indptr && ds && dh && dw_fold && db_fold && db_ih && dw_hh && db_hh,
               "ddfa_gru_step_bwd_image_v2: NULL pointer");
  DDFA_REQUIRE(dh != dh_out, "ddfa_gru_step_bwd_image_v2: dh must not alias dh_out");
  DDFA_REQUIRE(ds_prev == nullptr || (indptr_t && indices_t), "ddfa_gru_step_bwd_image_v2: ds_prev given without the transposed CSR");
  DDFA_REQUIRE(ds_prev == nullptr || ds_prev != ds, "ddfa_gru_step_bwd_image_v2: ds must not alias ds_prev");
  DDFA_REQUIRE(ds_prev == nullptr || ds_prev != dh, "ddfa_gru_step_bwd_image_v2: dh must not alias ds_prev");
  // moved by TMA bulk and tensor-map copies, which address 16-byte units
  DDFA_REQUIRE(aligned16(dh_out) && aligned16(ds) && aligned16(dh) && aligned16(gates_packed) && (h == nullptr || aligned16(h)),
               "ddfa_gru_step_bwd_image_v2: dh_out, ds, dh, gates_packed and h must be 16-byte aligned");
  return gru_tc2_step_bwd(dh_out, ds_prev, indptr_t, indices_t, h, h_image, s_image, nullptr, gates_packed, indptr, N, ds, dh, dw_fold, db_fold,
                          db_ih, dw_hh, db_hh, workspace, workspace_bytes, wgrad_mode, as_stream(stream_));
}

int ddfa_gru_step_bwd_finish(int32_t N, int32_t D, float *dw_fold, float *dw_hh, void *workspace, size_t workspace_bytes,
                             void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D == 128 && dw_fold && dw_hh, "ddfa_gru_step_bwd_finish: bad arguments (N=%d D=%d)", N, D);
  if (N == 0) return DDFA_OK;
  return gru_tc2_bwd_finish(N, dw_fold, dw_hh, workspace, workspace_bytes, as_stream(stream_));
}

int ddfa_gru_step_prepare_bwd(const float *w_fold, const float *w_hh, int32_t D, int engine, void *workspace,
                              size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  int rc = check_step_args("ddfa_gru_step_prepare_bwd", 0, D, engine);
  if (rc) return rc;
  if (engine == DDFA_ENGINE_SIMT) return DDFA_OK;
  DDFA_REQUIRE(w_fold && w_hh, "ddfa_gru_step_prepare_bwd: NULL pointer");
  if (D != 128) {      // the W' and Whh operand images at the head of the workspace (read K-major forward, MN-major here)
    if (workspace == nullptr || workspace_bytes < gru_tcw_weights_bytes(D)) {
      set_error("ddfa_gru_step_prepare_bwd: workspace too small (%zu < %zu)", workspace_bytes, gru_tcw_weights_bytes(D));
      return DDFA_ERR_WORKSPACE;
    }
    DDFA_REQUIRE(aligned16(w_fold) && aligned16(w_hh), "ddfa_gru_step_prepare_bwd: w_fold / w_hh not 16-byte aligned");
    return gru_tcw_prepare(w_fold, w_hh, D, workspace, as_stream(stream_));
  }
  return gru_tc2_prepare_bwd(w_fold, w_hh, workspace, workspace_bytes, as_stream(stream_));
}

int ddfa_gru_step_bwd(const float *dh_out, const float *h, const float *s, const float *gates, const int32_t *indptr,
                      const float *w_fold, const float *w_hh, int32_t N, int32_t D, float *ds, float *dh,
                      float *dw_fold, float *db_fold, float *db_ih, float *dw_hh, float *db_hh, void *workspace,
                      size_t workspace_bytes, int engine, void *stream_) {
  using namespace ddfa;
  int rc = check_step_args("ddfa_gru_step_bwd", N, D, engine);
  if (rc) return rc;
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(dh_out && h && s && gates && indptr && w_fold && w_hh && ds && dh && dw_fold && db_fold && db_ih && dw_hh && db_hh,
               "ddfa_gru_step_bwd: NULL pointer");
  DDFA_REQUIRE(dh != dh_out, "ddfa_gru_step_bwd: dh must not alias dh_out");
  cudaStream_t stream = as_stream(stream_);
  const size_t need = ddfa_gru_step_bwd_workspace_bytes(N, D, engine);
  if (workspace_bytes < need || workspace == nullptr) {
    set_error("ddfa_gru_step_bwd: workspace too small (%zu < %zu)", workspace_bytes, need);
    return DDFA_ERR_WORKSPACE;
  }
  if (engine == DDFA_ENGINE_TCGEN05 && D == 128) {
    // fp32-s convenience path (tests, tools): build the s image at the end of the workspace, then the image kernels
    void *s_img = gru_tc2_bwd_s_image_scratch(workspace, N);
    rc = act_to_image(s, N, s_img, stream);
    if (rc) return rc;
    return gru_tc2_step_bwd(dh_out, nullptr, nullptr, nullptr, h, /*h_img_in=*/nullptr, s_img, gates, nullptr, indptr, N, ds, dh, dw_fold, db_fold, db_ih, dw_hh, db_hh,
                            workspace, workspace_bytes, /*wgrad_mode=*/0, stream);
  }
  const bool wide = engine == DDFA_ENGINE_TCGEN05;       // D = 192 .. 512: tensor-core GEMMs, the rest as SIMT
  // wide: s and h become operand images through 16-byte loads, ds / dh are written with 8-byte stores
  DDFA_REQUIRE(!wide || (aligned16(s) && aligned16(h) && ((reinterpret_cast<uintptr_t>(ds) | reinterpret_cast<uintptr_t>(dh)) & 7) == 0),
               "ddfa_gru_step_bwd: s / h must be 16-byte aligned, ds / dh 8-byte aligned");
  float *dgi = reinterpret_cast<float *>(static_cast<uint8_t *>(workspace) + (wide ? gru_tcw_weights_bytes(D) : 0));
  float *dgh = dgi + (size_t)N * 3 * D;
  const bool det = deterministic();
  const int ctas = (N + kGateBwdRows - 1) / kGateBwdRows;
  float *bias_slots = dgh + (size_t)N * 3 * D;
  float *wg_part = bias_slots + (size_t)ctas * 7 * D;      // wide: the start of gru_tc_wide.cu's scratch
  dim3 block(D / 4, 256 / (D / 4) > 0 ? 256 / (D / 4) : 1);
  const size_t smem = sizeof(float) * block.y * 7 * D;
  gru_gate_bwd_kernel<<<ctas, block, smem, stream>>>(dh_out, h, gates, indptr, N, D, dgi, dgh, dh, db_fold, db_ih, db_hh,
                                                     det ? bias_slots : nullptr);
  DDFA_CHECK_LAUNCH("gru_gate_bwd_kernel");
  if (det) {
    bias_slots_sum_kernel<<<(7 * D + 255) / 256, 256, 0, stream>>>(bias_slots, ctas, D, db_fold, db_ih, db_hh);
    DDFA_CHECK_LAUNCH("bias_slots_sum_kernel");
  }
  if (wide) {
    return gru_tcw_bwd_gemms(dgi, dgh, s, h, N, D, workspace, wg_part, ds, dh, dw_fold, dw_hh, stream);
  }
  // ds = dgi @ w_fold ; dh = dh_out*z + dgh @ w_hh
  rc = sgemm(0, 0, N, D, 3 * D, 1.f, dgi, 3 * D, w_fold, D, 0.f, ds, D, 1, stream);
  if (rc) return rc;
  rc = sgemm(0, 0, N, D, 3 * D, 1.f, dgh, 3 * D, w_hh, D, 1.f, dh, D, 1, stream);
  if (rc) return rc;
  // dw_fold += dgi^T @ s ; dw_hh += dgh^T @ h   (K = N nodes -> split-K over the SMs; deterministic mode: slices added in order)
  const int split = simt_wgrad_split(N, D);
  if (det) {
    rc = sgemm_splitk_ordered(3 * D, D, N, 1.f, dgi, 3 * D, s, D, dw_fold, D, split, wg_part, stream);
    if (rc) return rc;
    return sgemm_splitk_ordered(3 * D, D, N, 1.f, dgh, 3 * D, h, D, dw_hh, D, split, wg_part, stream);
  }
  rc = sgemm(1, 0, 3 * D, D, N, 1.f, dgi, 3 * D, s, D, 1.f, dw_fold, D, split, stream);
  if (rc) return rc;
  rc = sgemm(1, 0, 3 * D, D, N, 1.f, dgh, 3 * D, h, D, 1.f, dw_hh, D, split, stream);
  return rc;
}

}  // extern "C"
