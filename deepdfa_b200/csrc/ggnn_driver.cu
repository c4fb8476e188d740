// Fused T-step drivers: the whole DGL GatedGraphConv forward / backward (reference: DDFA/code_gnn/models/flow_gnn/ggnn.py:57-60
// construction, :95 call -> dgl.nn.GatedGraphConv.forward: T x (linear, copy_u/sum message passing, GRUCell)) behind ONE C
// call each, for hosts that do not want to drive the per-step entry points themselves (SURVEY.md §8(b) export set).
// They only sequence the per-step entry points of this library — the same kernels, the same order deepdfa_b200/engine.py
// uses — and carve every intermediate out of ONE caller-provided workspace, which also carries the saved activations from
// ddfa_ggnn_fwd(training = 1) to ddfa_ggnn_bwd.
#include "common.cuh"

namespace ddfa {
namespace {

struct GgnnLayout {
  // offsets into the workspace (bytes); 0-sized regions are unused for the given mode
  size_t w_fold, b_fold, dw_fold, db_fold, gru_ws, h, h_img, s, gates, bwd_ws, ds, dh, total;
  size_t gru_ws_bytes, bwd_ws_bytes, plane, img, gate_step;
  int n_h, n_img, n_s;
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

GgnnLayout make_layout(int32_t N, int32_t D, int32_t T, int engine, int training) {
  GgnnLayout L = {};
  const bool tc = engine == DDFA_ENGINE_TCGEN05 && D == 128;     // the image path; at the wide widths tcgen05 keeps SIMT's layout
  L.plane = align256((size_t)N * D * sizeof(float));
  L.img = tc ? align256(ddfa_act_image_bytes(N)) : 0;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
  L.w_fold = take((size_t)3 * D * D * 4);
  L.b_fold = take((size_t)3 * D * 4);
  L.dw_fold = take((size_t)3 * D * D * 4);
  L.db_fold = take((size_t)3 * D * 4);
  L.gru_ws_bytes = ddfa_gru_step_workspace_bytes(tc ? 0 : N, D, engine);
  L.gru_ws = take(L.gru_ws_bytes < 16 ? 16 : L.gru_ws_bytes);
  // tcgen05: h_1 .. h_{T-1} exist only as activation images (no fp32 planes); the saved gates are packed 64-bit words (2 planes' worth)
  if (training) {
    L.n_h = (!tc && T > 1) ? T - 1 : 0;          // simt: h_1 .. h_{T-1} (h_0 = x and h_T = h_out belong to the caller)
    L.n_img = tc ? T : 0;                        // images of h_0 .. h_{T-1}
    L.n_s = T;                                   // s_0 .. s_{T-1}: images (tcgen05) or fp32 planes (simt)
  } else {
    L.n_h = (!tc && T > 1) ? 2 : 0;              // ping-pong
    L.n_img = tc ? 2 : 0;
    L.n_s = 1;
  }
  L.h = take((size_t)L.n_h * L.plane);
  L.h_img = take((size_t)L.n_img * L.img);
  L.s = take((size_t)L.n_s * (tc ? L.img : L.plane));
  if (training) {
    L.gate_step = tc ? align256(ddfa_gru_gates_packed_bytes(N, D)) : 4 * L.plane;
    L.gates = take((size_t)T * L.gate_step);
    L.bwd_ws_bytes = ddfa_gru_step_bwd_workspace_bytes_steps(N, D, engine, tc && T <= DDFA_WGRAD_MAX_STEPS ? T : 1);
    L.bwd_ws = take(L.bwd_ws_bytes < 16 ? 16 : L.bwd_ws_bytes);
    L.ds = take(2 * L.plane);
    L.dh = take(2 * L.plane);
  }
  L.total = off;
  return L;
}

inline float *f32_at(void *ws, size_t off) { return reinterpret_cast<float *>(static_cast<uint8_t *>(ws) + off); }
inline uint8_t *u8_at(void *ws, size_t off) { return static_cast<uint8_t *>(ws) + off; }

}  // namespace
}  // namespace ddfa

extern "C" {

size_t ddfa_ggnn_workspace_bytes(int32_t N, int32_t D, int32_t T, int engine, int training) {
  if (N < 0 || D <= 0 || T < 0) return 0;
  if (engine == DDFA_ENGINE_TCGEN05 && D != 128 && !ddfa::gru_tcw_width(D)) return 0;
  return ddfa::make_layout(N, D, T, engine, training).total;
}

#define GGNN_TRY(call)          \
  do {                          \
    const int rc__ = (call);    \
    if (rc__ != DDFA_OK) return rc__; \
  } while (0)

int ddfa_ggnn_fwd(const int32_t *indptr, const int32_t *indices, const float *x, int32_t N, int32_t D, int32_t T, const float *w_msg,
                  const float *b_msg, const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, float *h_out,
                  void *workspace, size_t workspace_bytes, int training, int engine, void *stream) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D > 0 && D % 4 == 0 && T >= 0, "ddfa_ggnn_fwd: bad sizes (N=%d D=%d T=%d)", N, D, T);
  DDFA_REQUIRE(engine == DDFA_ENGINE_SIMT || (engine == DDFA_ENGINE_TCGEN05 && (D == 128 || gru_tcw_width(D))),
               "ddfa_ggnn_fwd: the tcgen05 engine supports D = 128, 192, 256, 320, 384, 448 and 512 only (engine=%d D=%d)", engine, D);
  DDFA_REQUIRE(indptr && indices && x && w_msg && b_msg && w_ih && w_hh && b_ih && b_hh && h_out, "ddfa_ggnn_fwd: NULL pointer");
  DDFA_REQUIRE(h_out != x, "ddfa_ggnn_fwd: h_out must not alias x");
  const GgnnLayout L = make_layout(N, D, T, engine, training);
  if (workspace == nullptr || workspace_bytes < L.total) {
    set_error("ddfa_ggnn_fwd: workspace too small (%zu < %zu)", workspace_bytes, L.total);
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t cs = as_stream(stream);
  if (N == 0) return DDFA_OK;
  if (T == 0) {
    DDFA_CUDA(cudaMemcpyAsync(h_out, x, (size_t)N * D * sizeof(float), cudaMemcpyDeviceToDevice, cs));
    return DDFA_OK;
  }
  const bool tc = engine == DDFA_ENGINE_TCGEN05 && D == 128;
  float *w_fold = f32_at(workspace, L.w_fold), *b_fold = f32_at(workspace, L.b_fold);
  void *gws = u8_at(workspace, L.gru_ws);
  GGNN_TRY(ddfa_fold_weights_fwd(w_msg, b_msg, w_ih, D, w_fold, b_fold, stream));
  GGNN_TRY(ddfa_gru_step_prepare(w_fold, b_fold, b_ih, w_hh, b_hh, D, engine, gws, L.gru_ws_bytes, stream));
  auto h_buf = [&](int t) -> float * {     // storage of h_t for 1 <= t <= T-1
    return f32_at(workspace, L.h + (size_t)(training ? t - 1 : (t & 1)) * L.plane);
  };
  auto img_buf = [&](int t) { return u8_at(workspace, L.h_img + (size_t)(training ? t : (t & 1)) * L.img); };
  auto s_buf = [&](int t) { return u8_at(workspace, L.s + (size_t)(training ? t : 0) * (tc ? L.img : L.plane)); };
  if (tc) GGNN_TRY(ddfa_act_to_image(x, N, D, img_buf(0), stream));
  const float *h_cur = x;
  for (int t = 0; t < T; ++t) {
    float *g_t = training ? f32_at(workspace, L.gates + (size_t)t * L.gate_step) : nullptr;
    if (tc) {
      if (t == 0) GGNN_TRY(ddfa_gather_sum_image(indptr, indices, x, N, D, s_buf(t), nullptr, stream));
      else GGNN_TRY(ddfa_gather_sum_image_src(indptr, indices, img_buf(t), N, D, s_buf(t), stream));
      GGNN_TRY(ddfa_gru_step_fwd_image_v2(s_buf(t), img_buf(t), t == 0 ? x : nullptr, indptr, N, D, t == T - 1 ? h_out : nullptr,
                                          t + 1 < T ? img_buf(t + 1) : nullptr, g_t, gws, L.gru_ws_bytes, stream));
      continue;
    }
    float *h_next = (t == T - 1) ? h_out : h_buf(t + 1);
    {
      float *s_t = reinterpret_cast<float *>(s_buf(t));
      GGNN_TRY(ddfa_gather_sum(indptr, indices, h_cur, N, D, s_t, 0, stream));
      GGNN_TRY(ddfa_gru_step_fwd(s_t, h_cur, indptr, w_fold, b_fold, b_ih, w_hh, b_hh, N, D, h_next, g_t, gws, L.gru_ws_bytes, engine, stream));
    }
    h_cur = h_next;
  }
  return DDFA_OK;
}

int ddfa_ggnn_bwd(const int32_t *indptr, const int32_t *indptr_t, const int32_t *indices_t, const float *x, int32_t N, int32_t D, int32_t T,
                  const float *w_msg, const float *b_msg, const float *w_ih, const float *w_hh, const float *dh_T, float *dx,
                  float *dw_msg, float *db_msg, float *dw_ih, float *dw_hh, float *db_ih, float *db_hh, void *workspace,
                  size_t workspace_bytes, int engine, void *stream) {
  using namespace ddfa;
  DDFA_REQUIRE(N >= 0 && D > 0 && D % 4 == 0 && T >= 0, "ddfa_ggnn_bwd: bad sizes (N=%d D=%d T=%d)", N, D, T);
  DDFA_REQUIRE(engine == DDFA_ENGINE_SIMT || (engine == DDFA_ENGINE_TCGEN05 && (D == 128 || gru_tcw_width(D))),
               "ddfa_ggnn_bwd: the tcgen05 engine supports D = 128, 192, 256, 320, 384, 448 and 512 only (engine=%d D=%d)", engine, D);
  DDFA_REQUIRE(indptr && indptr_t && indices_t && x && w_msg && b_msg && w_ih && w_hh && dh_T && dx && dw_msg && db_msg && dw_ih && dw_hh &&
                   db_ih && db_hh,
               "ddfa_ggnn_bwd: NULL pointer");
  DDFA_REQUIRE(dx != dh_T, "ddfa_ggnn_bwd: dx must not alias dh_T");
  const GgnnLayout L = make_layout(N, D, T, engine, /*training=*/1);
  if (workspace == nullptr || workspace_bytes < L.total) {
    set_error("ddfa_ggnn_bwd: workspace too small (%zu < %zu)", workspace_bytes, L.total);
    return DDFA_ERR_WORKSPACE;
  }
  cudaStream_t cs = as_stream(stream);
  if (N == 0) return DDFA_OK;
  if (T == 0) {
    DDFA_CUDA(cudaMemcpyAsync(dx, dh_T, (size_t)N * D * sizeof(float), cudaMemcpyDeviceToDevice, cs));
    return DDFA_OK;
  }
  const bool tc = engine == DDFA_ENGINE_TCGEN05 && D == 128;
  const bool batched = tc && T <= DDFA_WGRAD_MAX_STEPS;
  float *w_fold = f32_at(workspace, L.w_fold);
  float *dw_fold = f32_at(workspace, L.dw_fold), *db_fold = f32_at(workspace, L.db_fold);
  void *bws = u8_at(workspace, L.bwd_ws);
  DDFA_CUDA(cudaMemsetAsync(dw_fold, 0, (size_t)3 * D * D * 4, cs));
  DDFA_CUDA(cudaMemsetAsync(db_fold, 0, (size_t)3 * D * 4, cs));
  GGNN_TRY(ddfa_gru_step_prepare_bwd(w_fold, w_hh, D, engine, bws, L.bwd_ws_bytes, stream));
  auto h_at = [&](int t) -> const float * { return t == 0 ? x : (tc ? nullptr : f32_at(workspace, L.h + (size_t)(t - 1) * L.plane)); };
  auto img_at = [&](int t) { return u8_at(workspace, L.h_img + (size_t)t * L.img); };
  auto s_at = [&](int t) { return u8_at(workspace, L.s + (size_t)t * (tc ? L.img : L.plane)); };
  float *ds_buf[2] = {f32_at(workspace, L.ds), f32_at(workspace, L.ds + L.plane)};
  float *dh_buf[2] = {f32_at(workspace, L.dh), f32_at(workspace, L.dh + L.plane)};
  const float *dh_in = dh_T;
  const float *ds_prev = nullptr;
  for (int t = T - 1; t >= 0; --t) {
    float *ds_t = ds_buf[t & 1];
    float *dh_t = (t == 0) ? dx : dh_buf[t & 1];          // the last step writes dL/dh_0 straight into dx
    const float *g_t = f32_at(workspace, L.gates + (size_t)t * L.gate_step);
    if (tc) {
      // incoming gradient = dh_in + A^T ds_prev: the transposed gather of the previous call's ds rides inside the call
      GGNN_TRY(ddfa_gru_step_bwd_image_v2(dh_in, ds_prev, indptr_t, indices_t, h_at(t), img_at(t), s_at(t), g_t, indptr, N, D, ds_t, dh_t,
                                          dw_fold, db_fold, db_ih, dw_hh, db_hh, bws, L.bwd_ws_bytes,
                                          batched ? DDFA_WGRAD_KEEP(t) : (t == T - 1 ? 1 : 2), stream));
      ds_prev = ds_t;
    } else {
      GGNN_TRY(ddfa_gru_step_bwd(dh_in, h_at(t), reinterpret_cast<const float *>(s_at(t)), g_t, indptr, w_fold, w_hh, N, D, ds_t, dh_t, dw_fold,
                                 db_fold, db_ih, dw_hh, db_hh, bws, L.bwd_ws_bytes, engine, stream));
      GGNN_TRY(ddfa_gather_sum(indptr_t, indices_t, ds_t, N, D, dh_t, 1, stream));      // dh_t += A^T ds_t
    }
    dh_in = dh_t;
  }
  if (tc) {
    GGNN_TRY(ddfa_gather_sum(indptr_t, indices_t, ds_prev, N, D, dx, 1, stream));        // the gather of the last ds (step 0)
    if (batched) {
      const void *s_imgs[DDFA_WGRAD_MAX_STEPS], *h_imgs[DDFA_WGRAD_MAX_STEPS];
      for (int t = 0; t < T; ++t) { s_imgs[t] = s_at(t); h_imgs[t] = img_at(t); }
      GGNN_TRY(ddfa_gru_bwd_wgrad_batched(s_imgs, h_imgs, T, N, D, dw_fold, dw_hh, bws, L.bwd_ws_bytes, stream));
    } else {
      GGNN_TRY(ddfa_gru_step_bwd_finish(N, D, dw_fold, dw_hh, bws, L.bwd_ws_bytes, stream));
    }
  }
  return ddfa_fold_weights_bwd(w_msg, b_msg, w_ih, dw_fold, db_fold, D, dw_msg, db_msg, dw_ih, stream);
}

}  // extern "C"
