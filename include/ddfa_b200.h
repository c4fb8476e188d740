/*
 * ddfa_b200.h — C ABI of libddfa_b200.so: the H100 (sm_90a) implementation of the DDFA
 * code_gnn GGNN hot path (embedding -> T x {edge gather-sum, GRU} -> attention readout -> MLP,
 * loss, backward, Adam).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter is documented "host";
 *   - tensors are dense, row-major, fp32 activations/parameters, int32 graph structure;
 *   - `stream` is a cudaStream_t passed as void*; every call only ENQUEUES work on it
 *     (no allocation, no synchronisation, CUDA-graph-capture safe);
 *   - return value: 0 on success, negative ddfa_status otherwise; ddfa_last_error()
 *     returns a thread-local message for the last failing call;
 *   - the caller owns all memory; workspace sizes are reported by *_workspace_bytes().
 *
 * Notation: N nodes, E edges (DGL orientation: message src -> dst, aggregated at dst),
 * B graphs, K embedding tables (1 or 4), H embedding width, D = K*H hidden width,
 * T propagation steps, L MLP layers, V vocabulary size.
 *
 * Each entry cites the reference interface it replaces (paths relative to the DeepDFA repo).
 */
#ifndef DDFA_B200_H
#define DDFA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DDFA_ABI_VERSION 1

typedef enum ddfa_status {
  DDFA_OK = 0,
  DDFA_ERR_INVALID_ARG = -1,   /* bad pointer / size / unsupported shape            */
  DDFA_ERR_CUDA = -2,          /* a CUDA runtime call or launch failed              */
  DDFA_ERR_UNSUPPORTED = -3,   /* shape outside what the selected engine supports   */
  DDFA_ERR_WORKSPACE = -4      /* workspace too small                               */
} ddfa_status;

/* GEMM engines for the dense GRU matmuls */
#define DDFA_ENGINE_SIMT 0     /* fp32 FFMA reference kernels (any D % 4 == 0)              */
#define DDFA_ENGINE_TCGEN05 1  /* tensor-core engine (name kept): Hopper wgmma, bf16x3 split operands, fp32 accumulate.
                                  D == 128: activation images, packed saved gates, fused backward (the entry points marked
                                  "tcgen05 engine" below).  D = 192, 256, 320, 384, 448, 512: the SIMT entry points' data flow
                                  (fp32 planes, fp32 saved gates) with tensor-core GEMMs (ddfa_gru_tc_wide_gemm).  Any other D:
                                  DDFA_ERR_UNSUPPORTED. */

int ddfa_abi_version(void);
const char *ddfa_last_error(void);
/* 1 if the current device is compute capability 10.x, 0 otherwise, <0 on CUDA error */
int ddfa_device_supported(void);
/* 1 if the given DDFA_ENGINE_* is compiled into this library, else 0 */
int ddfa_engine_available(int engine);
/* Tuning knobs: process-wide selectors between equivalent launch configurations of the same kernels (defaults compiled in;
 * the library reads no environment variables).  ddfa_tuning_get returns -1 for an unknown key. */
enum {
  DDFA_TUNE_L2_HINTS = 0,       /* bit mask of L2 eviction-priority hints, default 23 (csrc/common.cuh) */
  DDFA_TUNE_PDL_MASK = 1,       /* bit mask of kernels launched with programmatic stream serialization, default 15: 1 image gather, 2 forward GRU
                                   step, 4 the first kernel of a backward GRU step (the fused kernel, or the register-path gate backward),
                                   8 dgrad after the register-path gate backward */
  DDFA_TUNE_GATHER_VARIANT = 2, /* launch shape of the D = 128 edge gather (ddfa_gather_sum_variant ids), default 9 */
  DDFA_TUNE_FWD_PAIR = 3,       /* reserved: only 0 is accepted (the CTA-pair form of the forward kernel does not exist on sm_90a) */
  DDFA_TUNE_GATE_BWD_TMA = 4,   /* backward GRU step with the packed saved state: 0 register-path gate backward, then dgrad (two kernels, and the
                                   only path of the fp32 saved state); 1 one cluster kernel: gate backward on TMA-staged dh / gates / h, then dgrad;
                                   2 (default) = 1 + the folded gather's CSR scalars pipelined across tiles */
  DDFA_TUNE_GATHER_SRC_GROUPS = 5, /* image->image edge gather: row groups (of 4 rows) walked per warp with the CSR chain pipelined; 0 (default) = 1 group (2 / 4 measured neutral), or 1 / 2 / 4 */
  DDFA_TUNE_DETERMINISTIC = 6,  /* 0 (default): reductions may add float partial sums with atomics; 1: every reduction adds in a fixed order, so
                                   two runs with the same inputs, build, GPU model, shapes and tuning give bit-identical results.  Entry points
                                   without a deterministic form then fail with DDFA_ERR_INVALID_ARG / _UNSUPPORTED and a message naming the
                                   replacement: ddfa_embed_concat_bwd (use _ws), ddfa_readout_bwd (use _ws), ddfa_sgemm with split_k > 1.  ddfa_graph_label_bce[_valid] then needs
                                   `labels` whenever it computes the loss.  Like every key it is read when a call ENQUEUES its kernels: a
                                   captured CUDA graph keeps the kernels of the mode in force at capture time. */
  DDFA_TUNE__COUNT = 7
};
int ddfa_tuning_set(int key, int value);
int ddfa_tuning_get(int key);
/* development aid: in-kernel pipeline timeline of the tensor-core kernels (SM-clock stamps per CTA / tile / event, 132 x 12 x 12).
 * ddfa_debug_set(2, v): v = 0 off, 1 = forward + dgrad kernels, 2 = forward + wgrad kernels;
 * ddfa_debug_read(2 | 3, host, bytes): stamps of the backward (2) or forward (3) kernel's last launch;
 * ddfa_debug_read(4, host, 4): int32 count of timed-out mbarrier waits in the TMA-staged gather variants (0 when healthy);
 * ddfa_debug_read(5, host, 4): int32 number of 4-CTA clusters of the fused backward step kernel resident at once on this device. */
int ddfa_debug_set(int key, int value);
int ddfa_debug_read(int key, void *host_out, size_t bytes);
/* number of CUDA kernels this library has launched in this process (monotonic; for bench accounting) */
long long ddfa_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * Graph structure.  Replaces the DGLGraph the reference hands to GatedGraphConv / pooling
 * (DDFA/code_gnn/models/flow_gnn/ggnn.py:95,102; batches built by dgl.batch,
 * DDFA/sastvd/linevd/dataset.py:76, datamodule.py:116-141).
 * ------------------------------------------------------------------------------------- */

/* COO -> CSR-by-destination (indptr/indices: in-neighbours of each node, sorted by source id)
 * and CSR-by-source (indptr_t/indices_t: out-neighbours, sorted; the transposed graph used by
 * the backward gather).  src/dst are int64 (idx_bytes=8, what DGL hands over) or int32
 * (idx_bytes=4).  indptr, indptr_t: int32[N+1]; indices, indices_t: int32[E].
 * Either output pair may be NULL to skip it.  Returns DDFA_ERR_INVALID_ARG for N<0/E<0. */
size_t ddfa_build_csr_workspace_bytes(int64_t num_edges, int32_t num_nodes);
int ddfa_build_csr(const void *src, const void *dst, int idx_bytes, int64_t num_edges,
                   int32_t num_nodes, int32_t *indptr, int32_t *indices, int32_t *indptr_t,
                   int32_t *indices_t, void *workspace, size_t workspace_bytes, void *stream);

/* batch_num_nodes int64[B] (DGLGraph.batch_num_nodes()) -> graph_ptr int32[B+1] (exclusive scan). */
int ddfa_graph_ptr(const int64_t *batch_num_nodes, int32_t num_graphs, int32_t *graph_ptr,
                   void *stream);

/* Batch producer (SURVEY.md §8 f1): replaces the host-side collate — `dgl.batch([...])` in the GraphDataLoader
 * (DDFA/sastvd/linevd/datamodule.py:116-141) and `BigVulDatasetLineVD.get_indices` (DDFA/sastvd/linevd/dataset.py:63-76,
 * `dgl.batch([...]).to(device)`) — plus DGL's lazy CSR build, by slicing a device-resident ARENA of all graphs:
 *   arena = the CSR by destination and the CSR of the transposed graph over ALL graphs as one disjoint batch (what
 *   ddfa_build_csr produces for it), node_off int32[G+1] (first node of every graph), num_feats int64 feature vectors and
 *   the int32 _VULN vector over all nodes.
 * Out, for the graphs graph_ids[0..B) in that order: graph_ptr int32[B+1], indptr / indptr_t int32[N+1], indices /
 * indices_t int32[E], the feature vectors and _VULN restricted to the batch — bit-identical to ddfa_build_csr +
 * ddfa_graph_ptr on the collated COO of the same graphs.  batch_nodes / batch_edges = N and E of the batch (the caller
 * knows them from its host copy of the graph sizes; they size the outputs).  A bad id or inconsistent totals leave the
 * outputs untouched and raise the int32 counter at workspace[(B + 1) * 4]: its low 16 bits count bad ids, bit 16 flags
 * the totals.  Workspace layout (ddfa_arena_batch_workspace_bytes(B) bytes): int32 edge_ptr[B + 1] (first edge of every
 * graph of the batch, then E), int32 counter, int32 node_ptr[B + 1] (graph_ptr staged until the ids are known to be good).
 * feats / out_feats: host arrays of device pointers, num_feats <= 8. */
size_t ddfa_arena_batch_workspace_bytes(int32_t batch_size);
int ddfa_arena_batch(const int32_t *graph_ids, int32_t batch_size, int32_t num_graphs, const int32_t *node_off,
                     const int32_t *indptr, const int32_t *indices, const int32_t *indptr_t, const int32_t *indices_t,
                     const int64_t *const *feats, int32_t num_feats, const int32_t *vuln, int32_t batch_nodes,
                     int32_t batch_edges, int32_t *out_graph_ptr, int32_t *out_indptr, int32_t *out_indices,
                     int32_t *out_indptr_t, int32_t *out_indices_t, int64_t *const *out_feats, int32_t *out_vuln,
                     void *workspace, size_t workspace_bytes, void *stream);

/* Batch assembly from an encoder cache: the output of a FROZEN graph encoder (embedding + GatedGraphConv), computed once for
 * every node of an arena and kept as two fp32 planes h_all = h_T and x_all = the embedding rows, [num_nodes_all, D] each in
 * arena node order (node_off int32[num_graphs + 1] and vuln_all int32[num_nodes_all] as for ddfa_arena_batch).
 * Out, for the graphs graph_ids[0..B) in that order: graph_ptr int32[B+1], _VULN int32[N] and the rows of both planes,
 * out_h / out_x fp32 [N, D] — what the readout, the node head and their backward read.  No CSR is built and no edge is read.
 * batch_nodes = N, the batch's node total (the caller knows it from its host copy of the graph sizes).  Each graph's rows
 * are one contiguous slab per plane, cut into chunks of 128 float4 (2 KB per plane), one warp per chunk: a graph gets
 * ceil(n * D / 512) warps' worth of work, a 0-node graph none, so a large graph in a skewed batch is spread over as many
 * warps as its size needs.  Row offsets are 64-bit (a Big-Vul-size plane passes 2^32 bytes).  D: a positive multiple of 4;
 * h_all, x_all, out_h and out_x 16-byte aligned.  Output pointers may be NULL when N = 0.
 * Error contract of ddfa_arena_batch: a bad id (outside [0, num_graphs), or whose nodes lie outside [0, num_nodes_all)) or
 * a node total other than batch_nodes leaves every output untouched and raises the int32 counter at workspace[0]: its low
 * 16 bits count bad ids, bit 16 flags the total.  Only device words are read: the call is capturable.  Workspace layout
 * (ddfa_cache_batch_workspace_bytes(B) bytes): int32 counter, int32 node_ptr[B + 1] (graph_ptr staged until the ids are
 * known to be good), int32 chunk_ptr[B + 1] (each graph's first chunk).  A short workspace returns DDFA_ERR_WORKSPACE
 * before any launch. */
size_t ddfa_cache_batch_workspace_bytes(int32_t batch_size);
int ddfa_cache_batch(const int32_t *graph_ids, int32_t batch_size, int32_t num_graphs, const int32_t *node_off,
                     const int32_t *vuln_all, const float *h_all, const float *x_all, int32_t num_nodes_all, int32_t D,
                     int32_t batch_nodes, int32_t *out_graph_ptr, int32_t *out_vuln, float *out_h, float *out_x,
                     void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K1  embedding + concat.  Replaces ggnn.py:84-92 (4x nn.Embedding + torch.cat, or one).
 * idx[k]: int64[N] with values in [0,V); tables[k]: fp32[V,H]; x: fp32[N, K*H].
 * idx/tables are HOST arrays of K device pointers.  Out-of-range indices are clamped and
 * counted in *oob_count (int32 device counter, may be NULL) — the module raises on non-zero.
 * ------------------------------------------------------------------------------------- */
int ddfa_embed_concat_fwd(const int64_t *const *idx, const float *const *tables, int32_t num_tables,
                          int32_t vocab, int32_t width, int32_t num_nodes, float *x,
                          int32_t *oob_count, void *stream);
/* Same, and the rows also leave as h_0's activation image (row width K*H == 128; layout below, `image` holds
 * ddfa_act_image_bytes(num_nodes) bytes): what ddfa_act_to_image(x) would write, without the second pass over x.
 * Rows num_nodes .. (next multiple of 128) of the image are not written: the caller keeps them FINITE (e.g. zero-fills the
 * buffer once) — they are multiplied by the zero rows of the q images in the weight-gradient GEMM. */
int ddfa_embed_concat_fwd_image(const int64_t *const *idx, const float *const *tables, int32_t num_tables,
                                int32_t vocab, int32_t width, int32_t num_nodes, float *x, void *image,
                                int32_t *oob_count, void *stream);
/* dtables[k][idx_k[n], :] += (dx + dx2)[n, k*H:(k+1)*H]   (autograd of ggnn.py:84-92).
 * dx2 may be NULL; it lets the caller sum the two gradient paths into x (through the GGNN and
 * through the concat of ggnn.py:98) without a separate add kernel. */
int ddfa_embed_concat_bwd(const int64_t *const *idx, const float *dx, const float *dx2,
                          int32_t num_tables, int32_t vocab, int32_t width, int32_t num_nodes,
                          float *const *dtables, void *stream);
/* Same, with scratch for the deterministic form (DDFA_TUNE_DETERMINISTIC = 1: the nodes are sorted by index with a stable counting
 * sort and every table row is summed in node order, in fixed chunks).  workspace: ddfa_embed_concat_bwd_workspace_bytes(...)
 * bytes, 16-byte aligned; unused in the default mode. */
size_t ddfa_embed_concat_bwd_workspace_bytes(int32_t num_tables, int32_t vocab, int32_t width, int32_t num_nodes);
int ddfa_embed_concat_bwd_ws(const int64_t *const *idx, const float *dx, const float *dx2,
                             int32_t num_tables, int32_t vocab, int32_t width, int32_t num_nodes,
                             float *const *dtables, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K3  CSR edge gather-sum: out[v,:] = (accumulate ? out[v,:] : 0) + sum_{e in row v} h[indices[e],:]
 * Replaces DGL update_all(fn.copy_u('h','m'), fn.sum('m','a')) inside GatedGraphConv
 * (call site ggnn.py:95).  With the CSR-by-source arrays it is the backward of the same op.
 * D % 4 == 0, D <= 1024.  This is the HBM-roofline kernel (bytes: E*D*4 + N*D*4 + E*4 + (N+1)*4).
 * ------------------------------------------------------------------------------------- */
int ddfa_gather_sum(const int32_t *indptr, const int32_t *indices, const float *h,
                    int32_t num_nodes, int32_t dim, float *out, int accumulate, void *stream);
/* Tuning entry (scripts/gather_bench.py): same contract, explicit variant (D == 128): 0..9 register-path launch shapes,
 * 10 = neighbour rows staged in shared memory by per-row TMA bulk copies (cp.async.bulk + mbarrier), 11 = by tensor-map
 * tile::gather4 copies (four rows per UTMALDG) — csrc/gather_tma.cu. */
int ddfa_gather_sum_variant(int variant, const int32_t *indptr, const int32_t *indices, const float *h,
                            int32_t num_nodes, int32_t dim, float *out, int accumulate, void *stream);
/* The same gather for a source that exists only as its activation image (tcgen05 engine, steps t >= 1: h_t = hi + lo of the
 * image the forward GEMM read; no fp32 copy of h_t is kept).  D == 128. */
int ddfa_gather_sum_image_src(const int32_t *indptr, const int32_t *indices, const void *h_image,
                              int32_t num_nodes, int32_t dim, void *out_image, void *stream);


/* ---------------------------------------------------------------------------------------
 * Weight folding (done once per forward): w_fold = W_ih @ W  [3D,D], b_fold = W_ih @ b [3D]
 * so that  gi = (A h) w_fold^T + indeg * b_fold + b_ih  ==  GRUCell's  a W_ih^T + b_ih  with
 * a_v = sum_{u->v} (W h_u + b)   (DGL GatedGraphConv linears[0] + sum; ggnn.py:57-60).
 * ------------------------------------------------------------------------------------- */
int ddfa_fold_weights_fwd(const float *w_msg, const float *b_msg, const float *w_ih, int32_t dim,
                          float *w_fold, float *b_fold, void *stream);
/* dW_ih += dw_fold W^T + db_fold b^T ; dW += W_ih^T dw_fold ; db += W_ih^T db_fold */
int ddfa_fold_weights_bwd(const float *w_msg, const float *b_msg, const float *w_ih,
                          const float *dw_fold, const float *db_fold, int32_t dim, float *dw_msg,
                          float *db_msg, float *dw_ih, void *stream);

/* ---------------------------------------------------------------------------------------
 * K4  one GRU propagation step (torch.nn.GRUCell inside DGL GatedGraphConv; gate order r,z,n):
 *   gi = s w_fold^T + indeg b_fold + b_ih ; gh = h w_hh^T + b_hh
 *   r = sig(gi_r+gh_r) ; z = sig(gi_z+gh_z) ; n = tanh(gi_n + r*gh_n) ; h_out = (1-z)*n + z*h
 * s = gather-sum of h (K3).  indptr gives indeg.  If save_gates != NULL it receives
 * fp32[4][N][D] = r, z, n, gh_n (with b_hh_n) for the backward pass.
 * workspace: engine-dependent scratch (ddfa_gru_step_workspace_bytes).
 * ------------------------------------------------------------------------------------- */
size_t ddfa_gru_step_workspace_bytes(int32_t num_nodes, int32_t dim, int engine);
/* Once per forward (weights are constant over the T steps): engine-specific pre-packing of the
 * step's weights into `workspace` (tcgen05: bf16 hi/lo split, SWIZZLE_128B shared-memory operand images; SIMT:
 * no-op).  The same workspace must then be passed to every ddfa_gru_step_fwd of that forward. */
int ddfa_gru_step_prepare(const float *w_fold, const float *b_fold, const float *b_ih,
                          const float *w_hh, const float *b_hh, int32_t dim, int engine,
                          void *workspace, size_t workspace_bytes, void *stream);
int ddfa_gru_step_fwd(const float *s, const float *h, const int32_t *indptr, const float *w_fold,
                      const float *b_fold, const float *b_ih, const float *w_hh, const float *b_hh,
                      int32_t num_nodes, int32_t dim, float *h_out, float *save_gates,
                      void *workspace, size_t workspace_bytes, int engine, void *stream);
/* ---- tcgen05 engine: activation images -------------------------------------------------------
 * With the tcgen05 engine (D == 128) activations travel between kernels as MMA-ready operands next to /
 * instead of fp32: image[node/128][hi|lo][cols 0-63 | 64-127] = 16 KB chunks of [128 rows x 64 bf16] in the
 * UMMA K-major SWIZZLE_128B layout, hi = bf16(x), lo = bf16(x - hi); rows past N are zero; the image has
 * exactly the size of the fp32 matrix rounded up to 128 rows (ddfa_act_image_bytes).  Producers:
 * ddfa_act_to_image (from fp32, used for h_0 = x), ddfa_gather_sum_image (s_t), ddfa_gru_step_fwd_image
 * (h_{t+1}).  Allocate images zero-initialised. */
size_t ddfa_act_image_bytes(int64_t num_nodes);
int ddfa_act_to_image(const float *x, int32_t num_nodes, int32_t dim, void *image, void *stream);
/* K3 writing the image of s (and, when out_f32 != NULL, also the fp32 matrix). */
int ddfa_gather_sum_image(const int32_t *indptr, const int32_t *indices, const float *h,
                          int32_t num_nodes, int32_t dim, void *out_image, float *out_f32, void *stream);
/* K4 on images: s_image / h_image in, h (fp32, for the z*h term) in; h_out fp32 and (optional) its image out.
 * workspace = the buffer prepared by ddfa_gru_step_prepare(engine = TCGEN05). */
int ddfa_gru_step_fwd_image(const void *s_image, const void *h_image, const float *h,
                            const int32_t *indptr, int32_t num_nodes, int32_t dim, float *h_out,
                            void *h_out_image, float *save_gates, const void *workspace,
                            size_t workspace_bytes, void *stream);
/* The form the training / inference drivers use from round 2 on (fewer bytes per step, DESIGN.md §3):
 *   h            fp32 [N,128] or NULL — NULL: the z*h term takes h from h_image (h = hi + lo, 2^-17 relative);
 *   h_out        fp32 or NULL (only the last step needs it, for the readout); h_out_image or NULL; at least one of the two;
 *   save_gates_packed  NULL, or ddfa_gru_gates_packed_bytes(N, D) bytes: per element one 64-bit word — r, z as 14-bit,
 *                n as 16-bit fixed point, gh_n as a 20-bit float (csrc/tc_common.cuh: pack_gates; <= 3.1e-5 error) — the four
 *                saved gate values as ONE 8-byte store instead of four fp32 planes. */
size_t ddfa_gru_gates_packed_bytes(int32_t num_nodes, int32_t dim);
int ddfa_gru_step_fwd_image_v2(const void *s_image, const void *h_image, const float *h,
                               const int32_t *indptr, int32_t num_nodes, int32_t dim, float *h_out,
                               void *h_out_image, void *save_gates_packed, const void *workspace,
                               size_t workspace_bytes, void *stream);

/* Backward of one step on images (tcgen05 engine): like ddfa_gru_step_bwd below, but s arrives as its
 * activation image (the one ddfa_gather_sum_image wrote in the forward pass); the q matrices and h are turned
 * into images inside the workspace.  workspace: ddfa_gru_step_bwd_workspace_bytes(N, D, TCGEN05), prepared by
 * ddfa_gru_step_prepare_bwd. */
/* h_image: the image of h (step input) kept from the forward pass, or NULL (it is then rebuilt in the workspace).
 * ds_prev / indptr_t / indices_t: NULL, or the incoming gradient is dh_out + A^T ds_prev — the transposed edge gather
 * (autograd of ggnn.py:95's message sum) of the ds the NEXT time step's call produced is folded into this call, with
 * A^T given as the CSR of the transposed graph (ddfa_build_csr).  ds must not alias ds_prev. */
int ddfa_gru_step_bwd_image(const float *dh_out, const float *ds_prev, const int32_t *indptr_t, const int32_t *indices_t,
                            const float *h, const void *h_image, const void *s_image,
                            const float *gates, const int32_t *indptr, int32_t num_nodes, int32_t dim, float *ds, float *dh,
                            float *dw_fold, float *db_fold, float *db_ih, float *dw_hh, float *db_hh,
                            void *workspace, size_t workspace_bytes, int wgrad_mode, void *stream);
/* Same with the saved state of ddfa_gru_step_fwd_image_v2: gates_packed instead of four fp32 planes; h may be NULL
 * (then h_image, required here, supplies h = hi + lo). */
int ddfa_gru_step_bwd_image_v2(const float *dh_out, const float *ds_prev, const int32_t *indptr_t, const int32_t *indices_t,
                               const float *h, const void *h_image, const void *s_image,
                               const void *gates_packed, const int32_t *indptr, int32_t num_nodes, int32_t dim, float *ds, float *dh,
                               float *dw_fold, float *db_fold, float *db_ih, float *dw_hh, float *db_hh,
                               void *workspace, size_t workspace_bytes, int wgrad_mode, void *stream);
/* wgrad_mode: 0 = dw_fold / dw_hh are updated before the call returns (stream order); 1 / 2 = deferred: the
 * weight-gradient GEMM accumulates per-CTA partial sums inside the workspace over the T steps of one backward pass
 * (1 = first step, overwrites; 2 = later steps) and ddfa_gru_step_bwd_finish adds them to dw_fold / dw_hh once. */
int ddfa_gru_step_bwd_finish(int32_t num_nodes, int32_t dim, float *dw_fold, float *dw_hh, void *workspace,
                             size_t workspace_bytes, void *stream);
/* wgrad_mode = DDFA_WGRAD_KEEP(slot): run no weight-gradient GEMM in the step call; its q images stay in slot `slot` of a
 * workspace sized by ddfa_gru_step_bwd_workspace_bytes_steps(N, D, TCGEN05, steps).  After the last step ONE call does the
 * weight-gradient GEMM of all kept steps (K = steps x nodes) and adds it to dw_fold / dw_hh:
 * s_images / h_images = host arrays of `steps` device pointers, entry t = the images of s_t and h_t that belong to slot t. */
#define DDFA_WGRAD_KEEP(slot) (16 + (slot))
#define DDFA_WGRAD_MAX_STEPS 16
size_t ddfa_gru_step_bwd_workspace_bytes_steps(int32_t num_nodes, int32_t dim, int engine, int32_t steps);
int ddfa_gru_bwd_wgrad_batched(const void *const *s_images, const void *const *h_images, int32_t steps, int32_t num_nodes,
                               int32_t dim, float *dw_fold, float *dw_hh, void *workspace, size_t workspace_bytes, void *stream);

/* Backward of one step.  In: dh_out, h (step input), s, gates.  Out: ds [N,D] (to be
 * transposed-gathered by the caller), dh [N,D] = dh_out*z + dgh W_hh (overwritten).
 * Accumulated (+=): dw_fold[3D,D], db_fold[3D], db_ih[3D], dw_hh[3D,D], db_hh[3D].
 * workspace: ddfa_gru_step_bwd_workspace_bytes(); with the tcgen05 engine it must first be
 * prepared once per backward pass by ddfa_gru_step_prepare_bwd (transposed bf16 hi/lo weight
 * images) and is then reused by every step of that pass. */
size_t ddfa_gru_step_bwd_workspace_bytes(int32_t num_nodes, int32_t dim, int engine);
/* ddfa_gru_step_prepare / _prepare_bwd with engine = TCGEN05 at D = 192 .. 512 write the bf16 hi / lo operand images of W' and
 * Whh at the head of the step workspace; ddfa_gru_step_fwd / _bwd then run their GEMMs on the tensor cores (the images of the
 * step's activations are built inside the workspace).  The weight gradient is split over the nodes into slices that are added
 * in slice order in every mode (bit-identical on repeat). */
int ddfa_gru_step_prepare_bwd(const float *w_fold, const float *w_hh, int32_t dim, int engine,
                              void *workspace, size_t workspace_bytes, void *stream);
int ddfa_gru_step_bwd(const float *dh_out, const float *h, const float *s, const float *gates,
                      const int32_t *indptr, const float *w_fold, const float *w_hh,
                      int32_t num_nodes, int32_t dim, float *ds, float *dh, float *dw_fold,
                      float *db_fold, float *db_ih, float *dw_hh, float *db_hh, void *workspace,
                      size_t workspace_bytes, int engine, void *stream);
/* The tensor-core GEMMs of the step at the wide widths (D = 192 .. 512, D % 64 == 0), callable one by one (tests, tools); all
 * operands fp32 row-major, N = num_nodes rows:
 *   call 0: c[N,3D] = a[N,D] b[3D,D]^T      (gi = s W'^T, gh = h Whh^T)
 *   call 1: c[N,D] = a[N,3D] b[3D,D]        (ds = dgi W')
 *   call 2: c[N,D] += a[N,3D] b[3D,D]       (dh += dgh Whh)
 *   call 3: c[3D,D] += a[N,3D]^T b[N,D]     (dW' += dgi^T s, dWhh += dgh^T h; ddfa_gru_tc_wide_wgrad_slices(N, D) slices)
 * Rows of c past N are never written.  Other D: DDFA_ERR_UNSUPPORTED. */
size_t ddfa_gru_tc_wide_gemm_workspace_bytes(int call, int32_t num_nodes, int32_t dim);
int ddfa_gru_tc_wide_gemm(int call, const float *a, const float *b, int32_t num_nodes, int32_t dim, float *c, void *workspace,
                          size_t workspace_bytes, void *stream);
size_t ddfa_gru_tc_wide_wgrad_slices(int32_t num_nodes, int32_t dim);

/* ---------------------------------------------------------------------------------------
 * K3+K4 over all T steps: the whole dgl.nn.GatedGraphConv (ggnn.py:57-60 construction, :95 call) behind one call each.
 * They sequence the per-step entry points above (same kernels, same order as deepdfa_b200/engine.py) and carve every
 * intermediate out of ONE workspace of ddfa_ggnn_workspace_bytes(N, D, T, engine, training) bytes, which also carries
 * the saved activations from ddfa_ggnn_fwd(training = 1) to ddfa_ggnn_bwd (same workspace, untouched in between).
 *   fwd: x = h_0 [N,D] (the embedding output; must stay valid until the backward) -> h_out = h_T [N,D].
 *   bwd: dh_T [N,D] -> dx [N,D] = dL/dh_0 (overwritten); dw_msg[D,D], db_msg[D], dw_ih[3D,D], dw_hh[3D,D], db_ih[3D],
 *        db_hh[3D] accumulated (+=).  w_msg / b_msg = GatedGraphConv.linears[0], the rest = GatedGraphConv.gru.
 * engine = DDFA_ENGINE_SIMT (any D % 4 == 0) or DDFA_ENGINE_TCGEN05 (D = 128, 192, 256, 320, 384, 448, 512). */
size_t ddfa_ggnn_workspace_bytes(int32_t num_nodes, int32_t dim, int32_t n_steps, int engine, int training);
int ddfa_ggnn_fwd(const int32_t *indptr, const int32_t *indices, const float *x, int32_t num_nodes, int32_t dim,
                  int32_t n_steps, const float *w_msg, const float *b_msg, const float *w_ih, const float *w_hh,
                  const float *b_ih, const float *b_hh, float *h_out, void *workspace, size_t workspace_bytes,
                  int training, int engine, void *stream);
int ddfa_ggnn_bwd(const int32_t *indptr, const int32_t *indptr_t, const int32_t *indices_t, const float *x,
                  int32_t num_nodes, int32_t dim, int32_t n_steps, const float *w_msg, const float *b_msg,
                  const float *w_ih, const float *w_hh, const float *dh_T, float *dx, float *dw_msg, float *db_msg,
                  float *dw_ih, float *dw_hh, float *db_ih, float *db_hh, void *workspace, size_t workspace_bytes,
                  int engine, void *stream);

/* ---------------------------------------------------------------------------------------
 * K5-K7  readout + MLP.  Replaces torch.cat([ggnn_out, feat_embed]) (ggnn.py:98, never
 * materialised), DGL GlobalAttentionPooling(Linear(2D,1)) (ggnn.py:66-68,102) and the
 * output_layer MLP (ggnn.py:70-80,107).
 *   o_n = [h_T[n] | x[n]] ; g_n = <o_n, w_gate> + b_gate ; alpha = softmax of g over each graph
 *   pooled[b] = sum_n alpha_n o_n   (fp32[B,2D]; the encoder_mode output, ggnn.py:104-105)
 *   logits[b] = MLP(pooled[b])      (num_layers linears, ReLU between, last -> 1)
 * mlp_w / mlp_b: HOST arrays of num_layers device pointers ([2D,2D] ... [1,2D]); num_layers==0
 * skips the MLP (encoder mode; logits may be NULL).  Saved for backward when non-NULL:
 * gate_logit fp32[N], seg_max fp32[B], seg_sum fp32[B], mlp_act fp32[(L-1)][B][2D] (post-ReLU).
 * ------------------------------------------------------------------------------------- */
int ddfa_readout_mlp_fwd(const float *h_final, const float *x, const int32_t *graph_ptr,
                         int32_t num_graphs, int32_t dim, const float *w_gate, const float *b_gate,
                         const float *const *mlp_w, const float *const *mlp_b, int32_t num_layers,
                         float *pooled, float *logits, float *gate_logit, float *seg_max,
                         float *seg_sum, float *mlp_act, void *stream);
/* MLP backward: dlogits[B] -> dpooled[B,2D]; accumulates dmlp_w / dmlp_b (+=).
 * scratch: fp32[2][B][2D]. */
int ddfa_mlp_bwd(const float *dlogits, const float *pooled, const float *mlp_act,
                 const float *const *mlp_w, int32_t num_graphs, int32_t dim, int32_t num_layers,
                 float *dpooled, float *const *dmlp_w, float *const *dmlp_b, float *scratch,
                 void *stream);
/* MLP input gradient under DeepLift's rescale rule (captum DeepLift, the `nonlinear` rule at each nn.ReLU of the head):
 * dlogits[B] -> dpooled[B,2D], no weight or bias gradient.  pooled / mlp_act are the input pass's (as ddfa_readout_mlp_fwd wrote
 * them), pooled_ref / mlp_act_ref the reference (baseline) pass's.  At each hidden layer the pre-activations z, z' of both passes
 * are recomputed from the layer's inputs (one GEMM each) and the derivative [z > 0] is replaced by
 * (relu(z) - relu(z')) / (z - z'), or kept ([mlp_act > 0], the input pass's branch) where |z - z'| < 1e-10.  num_layers == 1: the
 * dpooled of ddfa_mlp_bwd.  mlp_b: HOST array of num_layers device pointers (read for layers < num_layers - 1).
 * scratch: fp32[4][B][2D]. */
int ddfa_mlp_dgrad_rescale(const float *dlogits, const float *pooled, const float *mlp_act, const float *pooled_ref,
                           const float *mlp_act_ref, const float *const *mlp_w, const float *const *mlp_b, int32_t num_graphs,
                           int32_t dim, int32_t num_layers, float *dpooled, float *scratch, void *stream);
/* Readout backward: dpooled[B,2D] -> dh_final[N,D], dx[N,D] (both overwritten);
 * accumulates dw_gate[2D], db_gate[1] (+=).  dpooled, pooled, h_final, x, w_gate, dh_final and dx
 * must be 16-byte aligned. */
int ddfa_readout_bwd(const float *dpooled, const float *pooled, const float *h_final, const float *x,
                     const int32_t *graph_ptr, int32_t num_graphs, int32_t dim, const float *w_gate,
                     const float *gate_logit, const float *seg_max, const float *seg_sum,
                     float *dh_final, float *dx, float *dw_gate, float *db_gate, void *stream);
/* Same, with scratch for the deterministic form (the graphs' dw_gate / db_gate terms added in graph order):
 * ddfa_readout_bwd_workspace_bytes(B, D) bytes; unused in the default mode.
 * dh_final == dx == NULL (this form only): the gate gradients alone, for an encoder whose parameters are frozen — h_final and x
 * are read once and no [N, D] plane is written; dw_gate / db_gate are bit-identical to the full call's in deterministic mode.
 * Exactly one of the two NULL is an error. */
size_t ddfa_readout_bwd_workspace_bytes(int32_t num_graphs, int32_t dim);
int ddfa_readout_bwd_ws(const float *dpooled, const float *pooled, const float *h_final, const float *x,
                        const int32_t *graph_ptr, int32_t num_graphs, int32_t dim, const float *w_gate,
                        const float *gate_logit, const float *seg_max, const float *seg_sum,
                        float *dh_final, float *dx, float *dw_gate, float *db_gate, void *workspace,
                        size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K8  graph labels + loss.  Replaces BaseModule.get_label (base_module.py:83-95: dgl.unbatch +
 * per-graph max of ndata["_VULN"]) and BCEWithLogitsLoss(pos_weight) (base_module.py:72-74,183).
 *   label[b] = max_n vuln[n] ; loss = (1/B) sum_b bce(logit_b, label_b; pos_weight)
 * dlogits[b] = grad_scale * d(sum_b bce)/dlogit_b  (caller passes grad_scale = 1/B_global).
 * loss_out: fp32[1] receives  loss_scale * sum_b bce  (caller passes loss_scale = 1/B_global).
 * vuln: int32[N].  labels: fp32[B] out.  dlogits may be NULL (evaluation).
 * ------------------------------------------------------------------------------------- */
int ddfa_graph_label_bce(const float *logits, const int32_t *vuln, const int32_t *graph_ptr,
                         int32_t num_graphs, float pos_weight, float loss_scale, float grad_scale,
                         float *labels, float *loss_out, float *dlogits, void *stream);
/* Same, for a batch padded to a bucket shape (FusedTrainer: one CUDA graph per bucket shape on a shuffled stream, the reference
 * reshuffles every epoch, datamodule.py:123-129): graphs [num_valid, num_graphs) are padding — they get a label but contribute
 * no loss term and dlogits = 0, so nothing of them reaches any gradient. */
int ddfa_graph_label_bce_valid(const float *logits, const int32_t *vuln, const int32_t *graph_ptr,
                               int32_t num_graphs, int32_t num_valid, float pos_weight, float loss_scale,
                               float grad_scale, float *labels, float *loss_out, float *dlogits, void *stream);

/* ---------------------------------------------------------------------------------------
 * K8'  label_style="node" loss (csrc/node_loss.cu): the rows the loss is taken over, drawn on the device, and the MLP head +
 * BCEWithLogits(pos_weight) over that row list.  Replaces BaseModule.resample (base_module.py:96-137: every vulnerable node plus
 * random.sample of round(n_vuln * factor) non-vulnerable ones) and the node-style loss (base_module.py:84-85,178-183).  Nothing
 * syncs with the host: num_nodes N is a CAPACITY that sizes every grid, the row count S lives in a device word, so one captured
 * CUDA graph serves every batch of a bucket shape.
 *
 * ddfa_node_sample: rows int32[N] receives the row list in ascending node order, *num_rows = S.
 *   Valid nodes are [0, *num_valid) (a device word: under shape bucketing the padding nodes are the tail).
 *   factor < 0 (no undersampling): every valid node; vuln / draw / status / workspace are not read (may be NULL).  One launch.
 *   factor >= 0: every valid node with vuln != 0, plus k = rint((double)n_vuln * factor) valid nodes with vuln == 0 drawn
 *   uniformly without replacement: the k smallest (key, node) pairs, key = word 0 of Philox4x32-10 with key `seed` and counter
 *   (draw lo, draw hi, node, 0).  *draw (int64 device word) is this call's draw index; the call advances it by one, so every
 *   replay of a captured launch draws afresh.  k larger than the population sets *status = 1 (never cleared by the call) and
 *   takes the whole population.  Launch sequence (fixed, 13 kernels + 1 memset): clear control words; count n_vuln and the
 *   population; k and the draw index; 4 x (key histogram of one 8-bit digit over the candidates, one-CTA bin pick) = radix
 *   select of the k-th smallest key, ties at it taken in node order; per-CTA counts; one-CTA scan in CTA order; write.
 *   Integer counts only: the rows do not depend on CTA scheduling.
 *   workspace: ddfa_node_sample_workspace_bytes(N) bytes, 4-byte aligned, scratch.
 * ddfa_node_head_fwd: for s < S, row r = rows[s]: o = [h_final[r] | x[r]] (read from the two fp32 [N, D] planes), num_layers
 *   linears with ReLU between (mlp_w / mlp_b as in ddfa_readout_mlp_fwd), logits[s] = the last output (fp32[N] capacity,
 *   compact).  mlp_act fp32[(L-1)][N][2D] receives the hidden activations (post-ReLU), compact: row s of layer i at
 *   mlp_act[(i*N + s)*2D].  SIMT fp32.
 * ddfa_node_bce: loss_out[0] = mean over s < S of bce(logits[s], (float)vuln[rows[s]]; pos_weight) (NaN for S = 0: a mean over
 *   nothing), dlogits[s] = its derivative (compact; may be NULL).  One CTA, a fixed summation order in both tuning modes.
 * ddfa_node_head_bwd: dlogits[S] -> dh_final, dx (fp32 [N, D] each, overwritten whole: zero outside the listed rows); accumulates
 *   (+=) dmlp_w / dmlp_b (host arrays of device pointers).  Weight and bias gradients are reduced over the rows in a fixed order
 *   in both tuning modes (32 private partials over fixed row chunks, added in chunk order): bit-reproducible.
 *   dh_final == dx == NULL: the weight and bias gradients alone (bit-identical to the full call's), for a frozen encoder; no
 *   [N, D] plane is written.  Exactly one of the two NULL is an error.
 *   workspace: ddfa_node_head_bwd_workspace_bytes(N, D) bytes, 16-byte aligned, scratch.
 * ------------------------------------------------------------------------------------- */
size_t ddfa_node_sample_workspace_bytes(int32_t num_nodes);
int ddfa_node_sample(const int32_t *vuln, const int32_t *num_valid, int32_t num_nodes, double factor, uint64_t seed,
                     int64_t *draw, int32_t *rows, int32_t *num_rows, int32_t *status, void *workspace,
                     size_t workspace_bytes, void *stream);
int ddfa_node_head_fwd(const float *h_final, const float *x, const int32_t *rows, const int32_t *num_rows,
                       int32_t num_nodes, int32_t dim, const float *const *mlp_w, const float *const *mlp_b,
                       int32_t num_layers, float *mlp_act, float *logits, void *stream);
int ddfa_node_bce(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows,
                  int32_t num_nodes, float pos_weight, float *loss_out, float *dlogits, void *stream);
/* ddfa_node_bce with dlogits[s] scaled by grad_scale: the row scale is (1.f / S) * grad_scale (gradient accumulation over k
 * micro-batches passes 1 / k).  loss_out is the unscaled mean; grad_scale = 1 gives results bit-identical to ddfa_node_bce. */
int ddfa_node_bce_scaled(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows,
                         int32_t num_nodes, float pos_weight, float grad_scale, float *loss_out, float *dlogits, void *stream);

/* Several ranks (data parallel): the draw ddfa_node_sample makes over the GLOBAL batch — the ranks' shards concatenated in rank
 * order — taken in phases, each rank keeping the rows that fall in its shard (local node ids).  Every phase reads and writes
 * device words only (capturable); between phases the caller runs an in-place int32 SUM all-reduce over the ranks of one region
 * of the rank's exchange buffer (ddfa_node_dp_exchange_words(world) int32 words):
 *   words [0, 256)                histogram of the current radix digit
 *   words [256, 256 + 2 world)    [n_vuln, n_nonvuln] of every rank (rank q writes its pair at 256 + 2q, the others are 0)
 *   words [256 + 2 world, + world) the ties at the threshold key of every rank (rank q writes word q)
 * Sequence (workspace: ddfa_node_sample_workspace_bytes(N), the same for every phase; num_valid as for ddfa_node_sample):
 *   ddfa_node_dp_count     clears the workspace's control words and the exchange buffer, counts this rank's valid vulnerable and
 *                          non-vulnerable nodes; factor < 0 also writes the local rows (every valid node) and *num_rows.
 *                          -> SUM the counts region.
 *   ddfa_node_dp_plan      global counts, *node_offset = sum over q < rank of rank q's valid nodes, *num_rows_global = S of the
 *                          global batch (n_vuln + k, or every valid node for factor < 0); factor >= 0: k, *status and *draw as
 *                          ddfa_node_sample computes them from the global counts (every rank advances its draw word alike).
 *                          factor < 0 ends here.
 *   4 x (ddfa_node_dp_radix_hist(pass) -> SUM the histogram region -> ddfa_node_dp_radix_pick(pass)): local histogram of the
 *                          keys' digit `pass`, bin pick on the global one.  Node n's key is that of node *node_offset + n of the
 *                          global batch: the keys one rank over the concatenated batch gives it.
 *   ddfa_node_dp_ties      per-CTA counts; this rank's ties at the threshold key into its tie word.  -> SUM the ties region.
 *   ddfa_node_dp_rows      the ties of ranks q < rank are taken first (global node order); compacts the local rows, *num_rows.
 * Integer counts only: the union over the ranks of node_offset + rows is ddfa_node_sample's row list of the global batch, bit
 * for bit, with the same status and draw.  One rank (world = 1, no exchange) is ddfa_node_sample itself.
 * ddfa_node_bce_global: ddfa_node_bce_scaled over this rank's S rows with the global row count *num_rows_global as the divisor:
 *   loss_out[0] = sum over the local rows of bce / S_global (this rank's share of the global mean; the shares of all ranks sum
 *   to it) and dlogits[s] = (1.f / S_global) * grad_scale * d bce (bit-identical to the one-rank rows' for the same S). */
size_t ddfa_node_dp_exchange_words(int32_t world);
int ddfa_node_dp_count(const int32_t *vuln, const int32_t *num_valid, int32_t num_nodes, double factor, int32_t rank,
                       int32_t world, int32_t *rows, int32_t *num_rows, void *workspace, size_t workspace_bytes,
                       int32_t *exchange, void *stream);
int ddfa_node_dp_plan(int32_t num_nodes, double factor, int32_t rank, int32_t world, int64_t *draw, int32_t *status,
                      int32_t *num_rows_global, int32_t *node_offset, void *workspace, size_t workspace_bytes,
                      const int32_t *exchange, void *stream);
int ddfa_node_dp_radix_hist(const int32_t *vuln, const int32_t *num_valid, int32_t num_nodes, uint64_t seed, int32_t pass,
                            void *workspace, size_t workspace_bytes, int32_t *exchange, void *stream);
int ddfa_node_dp_radix_pick(int32_t num_nodes, int32_t pass, void *workspace, size_t workspace_bytes, int32_t *exchange,
                            void *stream);
int ddfa_node_dp_ties(const int32_t *vuln, const int32_t *num_valid, int32_t num_nodes, uint64_t seed, int32_t rank,
                      int32_t world, void *workspace, size_t workspace_bytes, int32_t *exchange, void *stream);
int ddfa_node_dp_rows(const int32_t *vuln, const int32_t *num_valid, int32_t num_nodes, uint64_t seed, int32_t rank,
                      int32_t world, int32_t *rows, int32_t *num_rows, void *workspace, size_t workspace_bytes,
                      const int32_t *exchange, void *stream);
int ddfa_node_bce_global(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows,
                         const int32_t *num_rows_global, int32_t num_nodes, float pos_weight, float grad_scale,
                         float *loss_out, float *dlogits, void *stream);
size_t ddfa_node_head_bwd_workspace_bytes(int32_t num_nodes, int32_t dim);
int ddfa_node_head_bwd(const float *dlogits, const float *h_final, const float *x, const int32_t *rows,
                       const int32_t *num_rows, int32_t num_nodes, int32_t dim, const float *const *mlp_w,
                       int32_t num_layers, const float *mlp_act, float *dh_final, float *dx, float *const *dmlp_w,
                       float *const *dmlp_b, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K9  evaluation metrics accumulated on the device (csrc/eval_metrics.cu).  Replaces the torchmetrics bookkeeping of
 * BaseModule.validation_step (base_module.py:211-224: val_loss, Accuracy / Precision / Recall / F1Score of sigmoid(out)), of
 * test_step (base_module.py:238-323: the same metrics plus CatMetric test_preds / test_labels for the confusion matrix, the sklearn
 * report and the PR curve) and what the epoch ends compute from them (base_module.py:325-346).  One call adds one batch to a
 * persistent device METRIC STATE; nothing syncs with the host, so the launches can be captured into a CUDA graph.
 *
 * state: DDFA_EVAL_STATE_WORDS fp64 words, zero-initialised by the caller, 8-byte aligned:
 *   [0] TP  [1] FP  [2] TN  [3] FN  [4] samples  [5] batches  [6] sum_b loss_b * weight_b  [7] sum_b weight_b
 *   [8] predictions stored  [9] predictions dropped (overflow)  [10..15] reserved (left at zero)
 *   loss_b = the mean BCEWithLogits(pos_weight) over the batch's samples; a batch without samples adds no loss and no weight.
 *   Every count is an integer held exactly in fp64 (< 2^53), so states of several ranks add exactly (one all-reduce).
 * Per sample: x = logit, y = label (0 / 1), p = 1.f / (1.f + expf(-x)) (torch.sigmoid's expression), predicted positive iff
 *   p >= 0.5f — the binarisation of torchmetrics < 0.10, which val_* / test_* use.  The sklearn report of test_epoch_end uses
 *   p > 0.5; the two rules differ only at p == 0.5 exactly.  The BCE term is graph_label_bce's stable form, in fp32, summed in fp64.
 * Prediction store (probs_out / labels_out both NULL, or both fp32[capacity]): the batch's p and y go to positions
 *   state[8] + i (i = graph or row index), in input order; positions >= capacity are dropped and counted in state[9], the counts
 *   stay complete.
 * Order: per-CTA fp64 partials over a grid that depends on the capacity (num_graphs or num_nodes) only, added in CTA order by a
 *   second one-thread launch that also updates the state, in stream order: the state is bit-reproducible in both
 *   DDFA_TUNE_DETERMINISTIC modes.  Two launches per call.
 * weight: the batch's weight in the loss mean (finite, >= 0), by value.
 * workspace: ddfa_eval_metrics_workspace_bytes() bytes, 8-byte aligned, scratch.
 *
 * ddfa_eval_metrics_graph: label_style="graph".  Graph b < num_valid: y = max of vuln over [graph_ptr[b], graph_ptr[b+1]) (as
 *   ddfa_graph_label_bce), x = logits[b].  Graphs [num_valid, num_graphs) are bucket padding and are ignored.
 * ddfa_eval_metrics_rows: label_style="node".  Row s < S = *num_rows (a device word, clamped to [0, num_nodes]):
 *   x = logits[s] (compact, as ddfa_node_head_fwd writes them), y = vuln[rows[s]] (as ddfa_node_bce reads them).
 * ------------------------------------------------------------------------------------- */
#define DDFA_EVAL_STATE_WORDS 16
size_t ddfa_eval_metrics_workspace_bytes(void);
int ddfa_eval_metrics_graph(const float *logits, const int32_t *vuln, const int32_t *graph_ptr, int32_t num_graphs,
                            int32_t num_valid, float pos_weight, double weight, double *state, float *probs_out,
                            float *labels_out, int64_t capacity, void *workspace, size_t workspace_bytes, void *stream);
int ddfa_eval_metrics_rows(const float *logits, const int32_t *vuln, const int32_t *rows, const int32_t *num_rows,
                           int32_t num_nodes, float pos_weight, double weight, double *state, float *probs_out,
                           float *labels_out, int64_t capacity, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K9'  statement-level localisation (csrc/statements.cu): per-node scores of a batch and IVDetect's top-k statement metric
 * over them (DDFA/sastvd/helpers/evaluate.py:262-322, eval_statements_list), accumulated on the device like K9.
 *
 * ddfa_stmt_metric: function b < num_valid owns nodes [graph_ptr[b], graph_ptr[b+1]) (label_style="node": the function-level
 *   graph_ptr, not the one-node-per-graph view); functions [num_valid, num_graphs) are bucket padding and are ignored.  A function
 *   is vulnerable when one of its nodes has vuln != 0.  Its statements are ranked by score, descending, equal scores in node order
 *   (Python's stable sorted(..., reverse=True)); rank = the number of statements ahead of the first-ranked vulnerable one (the
 *   vulnerable node of maximum score, lowest node id among equal scores).  top-k is hit iff rank < k.
 *   state: DDFA_STMT_STATE_WORDS fp64 words, zero-initialised by the caller, 8-byte aligned, every word an integer count:
 *     [0] functions  [1] vulnerable functions  [2 + k - 1] vulnerable functions with rank < k, k = 1..10  [12] sum of rank over the
 *     vulnerable functions  [13] non-vulnerable functions without a score > threshold (DDFA_STMT_MODE_FULL only; the strict
 *     comparison of evaluate.py:276)  [14] functions with a NaN score (counted here and in [0] only)  [15] batches
 *   One CTA per function (grid-stride over a grid of min(num_graphs, 264) CTAs), two passes over its nodes, integer partials per
 *   CTA added in CTA order by a second one-thread launch: the state is bit-reproducible in both DDFA_TUNE_DETERMINISTIC modes.
 *   workspace: ddfa_stmt_metric_workspace_bytes() bytes, 8-byte aligned, scratch.  Two launches.
 * ddfa_stmt_attention: alpha[n] = exp(gate_logit[n] - seg_max[b]) / seg_sum[b] for the nodes of every graph b < num_graphs — the
 *   softmax gate of GlobalAttentionPooling (DGL's get_attention=True) from the three arrays ddfa_readout_mlp_fwd writes when given,
 *   with the expression of ddfa_readout_bwd.  One launch.
 * ddfa_stmt_input_grad_score: score[n] = weight * sum_d f(x, g)[n, d] (accumulate != 0: score[n] = fmaf(weight, sum, score[n])), with
 *   g = dh + dx ([N, dim] each: the gradient of h_0 through the GGNN and of the direct use of x in the readout concat, which
 *   the embedding backward would add) and f = |g| (DDFA_STMT_SCORE_ABS; x may be NULL) or x * g (DDFA_STMT_SCORE_X_TIMES).  Warp
 *   per node, a fixed shuffle tree: bit-reproducible.  One launch.
 * ddfa_stmt_scale_input: out = alpha * x (fp32 [N, dim], out must not alias x) and, when image != NULL (dim == 128), its
 *   activation image as ddfa_act_to_image writes it: the start of a forward from a scaled embedding output.  One or two launches.
 * ddfa_stmt_node_probability: scores[n] = 1.f / (1.f + expf(-logits[n])) for n < S = *num_rows (clamped to [0, num_nodes]), 0
 *   beyond: the probabilities of ddfa_eval_metrics_rows when the rows are every valid node in order.  One launch.
 * ddfa_stmt_attribution_score: score[n] = weight * sum_d diff[n, d] * (dh + dx)[n, d] (accumulate != 0: fmaf(weight, sum,
 *   score[n])): the DDFA_STMT_SCORE_X_TIMES rule of ddfa_stmt_input_grad_score over a given difference tensor (x - baseline), the
 *   same sums bit for bit.  One launch.
 * ddfa_stmt_shap_input: the input of one DeepLift / GradientShap pass.  Per function b < num_graphs (nodes [graph_ptr[b],
 *   graph_ptr[b+1])) and element (n, d): x~ = x + noise_stdev * eps, base = baseline_stdev * eps', diff = x~ - base and
 *   input = fmaf(a_b, diff, base), with a_b = alpha when alpha >= 0 (0: the baseline itself) and otherwise drawn uniform in [0, 1).
 *   The draws are Philox4x32-10 with key `seed` and counter (c0, c1, c2, c3) = (low word of *counter, sample, index, column
 *   word): a_b = (w0 >> 8) * 2^-24 of (batch, sample, b, 0x80000000); eps of columns 4q..4q+3 of node n from the words of
 *   (batch, sample, n, q) — for eps', q | 0x40000000 — by Box-Muller on the pairs (w0, w1), (w2, w3): r = sqrt(-2 ln u1),
 *   u1 = ((w_a >> 8) + 1) 2^-24, u2 = (w_b >> 8) 2^-24, (r cos 2 pi u2, r sin 2 pi u2).  A stdev of 0 draws nothing.  *counter
 *   (int64, device) is read, not advanced.  dim % 4 == 0; x, input and diff fp32 [N, dim], 16-byte aligned, not aliased.  When
 *   image != NULL (dim == 128) input is also written as its activation image (ddfa_act_to_image).  One or two launches.
 * ------------------------------------------------------------------------------------- */
#define DDFA_STMT_STATE_WORDS 16
#define DDFA_STMT_MODE_VULN_ONLY 0
#define DDFA_STMT_MODE_FULL 1
#define DDFA_STMT_SCORE_ABS 0
#define DDFA_STMT_SCORE_X_TIMES 1
size_t ddfa_stmt_metric_workspace_bytes(void);
int ddfa_stmt_metric(const float *scores, const int32_t *vuln, const int32_t *graph_ptr, int32_t num_graphs, int32_t num_valid,
                     int32_t mode, float threshold, double *state, void *workspace, size_t workspace_bytes, void *stream);
int ddfa_stmt_attention(const float *gate_logit, const float *seg_max, const float *seg_sum, const int32_t *graph_ptr,
                        int32_t num_graphs, float *alpha, void *stream);
int ddfa_stmt_input_grad_score(const float *x, const float *dh, const float *dx, int32_t num_nodes, int32_t dim, int32_t rule,
                               float weight, int32_t accumulate, float *score, void *stream);
int ddfa_stmt_scale_input(const float *x, float alpha, int32_t num_nodes, int32_t dim, float *out, void *image, void *stream);
int ddfa_stmt_node_probability(const float *logits, const int32_t *num_rows, int32_t num_nodes, float *scores, void *stream);
int ddfa_stmt_attribution_score(const float *diff, const float *dh, const float *dx, int32_t num_nodes, int32_t dim, float weight,
                                int32_t accumulate, float *score, void *stream);
int ddfa_stmt_shap_input(const float *x, const int32_t *graph_ptr, int32_t num_graphs, int32_t num_nodes, int32_t dim, float alpha,
                         float noise_stdev, float baseline_stdev, uint64_t seed, const int64_t *counter, int32_t sample, float *input,
                         float *diff, void *image, void *stream);

/* ---------------------------------------------------------------------------------------
 * K9''  prediction store (csrc/predict.cu): per function of a batch, its probability, its DDFA embedding and its top-k
 * statements, appended to a device result store at a device cursor.  Nothing is read from the host, so the call can be
 * captured into a CUDA graph and every replay appends.
 *
 * ddfa_predict_store: function b < num_valid owns nodes [graph_ptr[b], graph_ptr[b+1]) (int32 [num_graphs + 1]; label_style="node":
 *   the function-level graph_ptr) and goes to store position p = cursor[0] + b, cursor[0] read on the device.  Positions
 *   >= capacity are dropped and counted in cursor[1]; cursor[0] advances by the number stored.  Functions [num_valid, num_graphs)
 *   are bucket padding and are ignored.  cursor: int64[2] on the device, [0] stored, [1] dropped, 8-byte aligned.
 *   prob_out (fp32 [capacity]), given exactly when logits or node_probs is (never both):
 *     logits (graph style, fp32 [num_graphs]): prob_out[p] = 1.f / (1.f + expf(-logits[b])), the p of ddfa_eval_metrics_*;
 *     node_probs (node style, fp32 per node): the maximum over the function's nodes (a function is flagged when any statement is,
 *     evaluate.py:276); a NaN among them gives NaN, a function without nodes 0.
 *   emb_out (fp32 [capacity, out_dim]), given exactly when pooled (fp32 [num_graphs, out_dim]) is: emb_out[p, :] = pooled[b, :].
 *   top_idx_out (int32 [capacity, k]) / top_score_out (fp32 [capacity, k]), given with scores (fp32 per node) exactly when k > 0,
 *     0 <= k <= DDFA_PREDICT_MAX_K: rank j's node index local to the function (n - graph_ptr[b]) and its raw score.  The ranking
 *     is ddfa_stmt_metric's: score descending, equal scores (-0.0 == +0.0) in node order (Python's stable sorted(...,
 *     reverse=True)); NaN ranks after every number, -inf included, NaNs in node order.  Ranks j >= the function's node count
 *     get -1 and NaN.
 *   One CTA per function (grid-stride over min(num_graphs, 264) CTAs), min(k, nodes) selection rounds over its scores, each
 *   the maximum of a unique 64-bit (score, node) key below the previous round's: exact, no atomics, bit-reproducible in both
 *   DDFA_TUNE_DETERMINISTIC modes, correct for any segment length.  Two launches (the second advances the cursor), none when
 *   num_valid == 0.
 * ------------------------------------------------------------------------------------- */
#define DDFA_PREDICT_MAX_K 32
int ddfa_predict_store(const float *logits, const float *node_probs, const float *pooled, int32_t out_dim, const float *scores,
                       int32_t k, const int32_t *graph_ptr, int32_t num_graphs, int32_t num_valid, float *prob_out,
                       float *emb_out, int32_t *top_idx_out, float *top_score_out, int64_t *cursor, int64_t capacity,
                       void *stream);

/* ---------------------------------------------------------------------------------------
 * K9'''  threshold curves of a test pass (csrc/curves.cu): what BaseModule.test_epoch_end (base_module.py:348-383) computes from
 * test_preds / test_labels with torchmetrics < 0.10 — the exact precision-recall curve, the binned one — plus the ROC curve,
 * AUROC and average precision, over n fp32 probabilities and n fp32 labels (the layout of the K9 prediction store).  Nothing
 * syncs with the host: the curve lengths go to device words.
 *
 * ddfa_curve_sort: torchmetrics' _binary_clf_curve.  The probabilities sorted in descending order (an LSD radix sort of 8-bit
 *   digits over the 32-bit order-preserving key of p; -0.0 is keyed as +0.0, as the reference ties them); at the last sample of
 *   every run of equal values, in descending order j = 0 .. m-1: thresholds[j] = the value (the stored fp32 bits; +0.0 for a
 *   zero), tps[j] / fps[j] = the samples with p >= thresholds[j] whose label is 1 / is not.  thresholds fp32 [n], tps / fps
 *   int64 [n]; entries j >= m are not written.
 * info: DDFA_CURVE_INFO_WORDS int64 words, 8-byte aligned, zeroed and filled by ddfa_curve_sort, read (and [1] written) by
 *   ddfa_curve_metrics:
 *   [0] m, distinct thresholds  [1] PR curve points before the appended (1, 0)  [2] positives (label == 1)  [3] negatives
 *   [4] NaN probabilities  [5] labels other than 0 / 1 (NaN included; they count as negatives)  [6] 1 when only one class is
 *   present (no positive or no negative: the ROC curve and AUROC are undefined)  [7] reserved
 *   The outputs are computed whatever the error words say (never a fault); with [4] > 0 they follow the key order of NaN and are
 *   meaningless.
 * ddfa_curve_metrics (over ddfa_curve_sort's outputs; P = info[2], N = info[3], L = info[1]):
 *   PR curve, torchmetrics < 0.10's _precision_recall_curve_compute_single_class: truncated at the first j where tps[j] == P
 *     (L = j + 1 points), reversed, then precision 1 / recall 0 appended: pr_precision / pr_recall fp64 [n + 1] (L + 1 written),
 *     pr_thresholds fp32 [n] (L written): for k < L, q = L - 1 - k: tps[q] / (tps[q] + fps[q]), tps[q] / P, thresholds[q].
 *   ROC curve, _roc_compute_single_class: a leading (0, 0) point at thresholds[0] + 1.f, then fpr = fps / N, tpr = tps / P (0
 *     where N or P is 0): roc_fpr / roc_tpr fp64 [n + 1], roc_thresholds fp32 [n + 1] (m + 1 written).
 *   summary fp64 [2]: [0] AUROC = sum over the ROC points of (fpr[j+1] - fpr[j]) * (tpr[j] + tpr[j+1]) / 2 (NaN with one class),
 *     [1] average precision = -sum over the PR points of (recall[k+1] - recall[k]) * precision[k] (NaN without positives).  fp64
 *     terms, per-CTA partials over a grid that depends on n only, added in CTA order: bit-reproducible in both
 *     DDFA_TUNE_DETERMINISTIC modes.
 *   Binned curve, BinnedPrecisionRecallCurve: for the fp32 thresholds bin_thresholds[0 .. num_bins), TP / FP = the samples with
 *     p >= t_i by label (binary search over thresholds), FN = P - TP; bin_precision[i] = (TP + 1e-6) / (TP + FP + 1e-6),
 *     bin_recall[i] = TP / (TP + FN + 1e-6) in fp64, then 1 / 0 at [num_bins]: fp64 [num_bins + 1] each.
 * workspace: ddfa_curve_workspace_bytes(n) bytes, 16-byte aligned, scratch; one buffer serves both calls.  Every entry runs on
 *   `stream` and can be captured.  ddfa_curve_sort: 1 memset + 16 launches; ddfa_curve_metrics: 3 launches.  1 <= n.
 * ------------------------------------------------------------------------------------- */
#define DDFA_CURVE_INFO_WORDS 8
size_t ddfa_curve_workspace_bytes(int64_t n);
int ddfa_curve_sort(const float *probs, const float *labels, int64_t n, float *thresholds, int64_t *tps, int64_t *fps,
                    int64_t *info, void *workspace, size_t workspace_bytes, void *stream);
int ddfa_curve_metrics(const float *thresholds, const int64_t *tps, const int64_t *fps, int64_t n, const float *bin_thresholds,
                       int32_t num_bins, double *pr_precision, double *pr_recall, float *pr_thresholds, double *roc_fpr,
                       double *roc_tpr, float *roc_thresholds, double *bin_precision, double *bin_recall, double *summary,
                       int64_t *info, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K10  torch.optim.Adam(lr, betas, eps, weight_decay) with coupled L2 (DDFA/configs/
 * config_default.yaml:43-47) over one flat parameter buffer.  step_count: int32[1] device
 * counter, incremented by the kernel (graph-capture safe).
 * ------------------------------------------------------------------------------------- */
int ddfa_adam_flat(float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                   int32_t *step_count, int64_t numel, float lr, float beta1, float beta2, float eps,
                   float weight_decay, void *stream);
/* Same kernel, hyperparameters from device memory: hyper = 5 device floats [lr, beta1, beta2, eps, weight_decay].
 * The words are read when the kernel RUNS, not when it is enqueued: a launch captured into a CUDA graph uses whatever
 * the words hold at each replay, so a learning-rate schedule reaches captured steps (write the words in stream order
 * before the replay).  Equal values give bit-identical parameters and moments to ddfa_adam_flat. */
int ddfa_adam_flat_hp(float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                      int32_t *step_count, int64_t numel, const float *hyper, void *stream);
/* The update over the trainable elements of a partly frozen model: ranges = device int64[2 * num_ranges], sorted, disjoint
 * [begin, end) pairs inside [0, numel), every bound a multiple of 4.  Elements outside the ranges are neither read nor written
 * (parameters and both moments stay bit-unchanged); inside, results are bit-identical to ddfa_adam_flat_hp (gstate == NULL) or
 * ddfa_adam_flat_guarded (gstate != NULL, skipped as there) on the same elements.  step_count advances once per call (not on a
 * skipped step), also when num_ranges == 0. */
int ddfa_adam_flat_ranges(float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                          int32_t *step_count, int64_t numel, const int64_t *ranges, int32_t num_ranges,
                          const float *hyper, const float *gstate, int32_t *skipped, void *stream);
/* Parameter groups: torch.optim.Adam / torch.optim.AdamW (Adam(decoupled_weight_decay=True)) with several param_groups.
 *   groups = device fp32[num_groups * DDFA_ADAM_GROUP_WORDS], one row per group:
 *            [lr, beta1, beta2, eps, weight_decay, decoupled (1.0f / 0.0f), decay, pad], 1 <= num_groups <= DDFA_ADAM_MAX_GROUPS,
 *            read when the kernel RUNS (as hyper in ddfa_adam_flat_hp).  decay = (float)(1.0 - (double)lr * weight_decay),
 *            computed in double and rounded once, as torch's Python scalar is; coupled groups ignore it.
 *   ranges = device int64[3 * num_ranges], sorted, disjoint [begin, end, group] triples inside [0, numel), every bound a
 *            multiple of 4, group in [0, num_groups).  Elements outside every range are neither read nor written.
 * A coupled group (decoupled = 0) computes torch.optim.Adam: results bit-identical to ddfa_adam_flat_ranges with that row's
 * first five words as hyper.  A decoupled group computes torch.optim.AdamW's order (torch/optim/adam.py, _single_tensor_adam):
 * p *= decay first, then the same moment and step expressions with no weight_decay * p term in the gradient.  Bias
 * corrections are per group (fp64, from the one step_count).  gstate / skipped: NULL, or the guard as in ddfa_adam_flat_guarded.
 * step_count advances once per call (not on a skipped step), also when num_ranges == 0. */
#define DDFA_ADAM_GROUP_WORDS 8
#define DDFA_ADAM_MAX_GROUPS 64
int ddfa_adam_flat_groups(float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                          int32_t *step_count, int64_t numel, const int64_t *ranges, int32_t num_ranges,
                          const float *groups, int32_t num_groups, const float *gstate, int32_t *skipped, void *stream);

/* ---------------------------------------------------------------------------------------
 * K10'  The data-parallel exchange fused with the optimizer over NVLink peer memory: ONE kernel per rank does
 * reduce-scatter (16-byte loads from every peer's gradient buffer) + Adam with coupled L2 on the rank's 1/R slice (moments are
 * sharded: exp_avg / exp_avg_sq are touched only inside the slice) + all-gather (16-byte stores of the new parameters into every
 * peer's parameter buffer), bracketed by two flag barriers in peer memory (csrc/allreduce_adam.cu).  Replaces
 * ncclAllReduce(flat gradients) + ddfa_adam_flat on every rank.  Collective: every rank launches it once per step.
 *   peer_params / peer_grads / peer_flags: HOST arrays of `world` device pointers, entry p = rank p's buffer as addressable from
 *   this device (symmetric allocation, peer-mapped); flags: >= 2 * world uint32 per rank, zero-initialised once;
 *   numel % 4 == 0; loss_offset: element index inside the gradient buffers of the per-rank loss word (summed into *loss_out,
 *   a LOCAL word; may be NULL); ticket: one zero-initialised local uint32; step_count as in ddfa_adam_flat (read as the
 *   barrier epoch, then incremented).  CUDA-graph capturable; waits are bounded (trap, not hang).
 * ------------------------------------------------------------------------------------- */
int ddfa_allreduce_adam_p2p(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                            int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                            int64_t numel, int64_t loss_offset, float *loss_out, uint32_t *ticket, float lr,
                            float beta1, float beta2, float eps, float weight_decay, void *stream);
/* Same protocol, hyperparameters from device memory: hyper = 5 LOCAL device floats [lr, beta1, beta2, eps, weight_decay],
 * read when the kernel runs (as in ddfa_adam_flat_hp: captured launches see later writes).  Every rank must hold the same
 * values.  The owner of element i is rank floor(i / 4 / per), per = ceil(numel / 4 / world): only the owner reads and
 * writes exp_avg / exp_avg_sq there. */
int ddfa_allreduce_adam_p2p_hp(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                               int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                               int64_t numel, int64_t loss_offset, float *loss_out, uint32_t *ticket,
                               const float *hyper, void *stream);

/* ---------------------------------------------------------------------------------------
 * Gradient guard: torch.nn.utils.clip_grad_norm_(params, max_norm, norm_type=2) between the gradient exchange and Adam,
 * and GradScaler's rule for a non-finite step (optimizer.step() is not called), inside the (capturable) optimizer step.
 *   norm = sqrt(sum g^2): squares summed in fp64 in a fixed order (the same in both DDFA_TUNE_DETERMINISTIC modes), rounded
 *          once to fp32.  torch sums in fp32 and returns inf once an element exceeds ~1e19; here every finite gradient gives a
 *          finite norm unless the norm itself exceeds FLT_MAX.
 *   coef = min(1, max_norm / (norm + 1e-6)) in fp32, as torch computes it; Adam uses g * coef where it used g (before the
 *          coupled L2 term).  coef == 1 (max_norm = +inf, or a norm below the bound) gives results bit-identical to the
 *          unguarded entry points.
 *   skip: with `skipped` != NULL, a step whose norm is not finite writes no parameter, no moment and not the step counter,
 *          and adds 1 to *skipped (int32 device counter).  With skipped == NULL a non-finite norm is not special: coef is
 *          then NaN or 0 and flows into the update, as in torch.
 * gstate: 3 device floats [norm, coef, nonfinite (1.0f / 0.0f)], written by the norm computation.
 * max_norm: NULL (no clipping) or ONE device float read when the kernel runs, so a captured launch sees later writes; +inf
 * measures without clipping.
 * ------------------------------------------------------------------------------------- */
size_t ddfa_grad_norm_workspace_bytes(int64_t numel);
/* The norm of grads[0, numel) (a fixed grid of fp64 per-CTA partials, added in CTA order by a second launch) -> gstate.
 * workspace: ddfa_grad_norm_workspace_bytes(numel) bytes, 8-byte aligned, scratch. */
int ddfa_grad_norm(const float *grads, int64_t numel, const float *max_norm, float *gstate, void *workspace,
                   size_t workspace_bytes, void *stream);
/* ddfa_adam_flat_hp with the clipped gradient g * gstate[1]; skipped as above (the step-counter increment reads the flag too). */
int ddfa_adam_flat_guarded(float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                           int32_t *step_count, int64_t numel, const float *hyper, const float *gstate,
                           int32_t *skipped, void *stream);
/* ddfa_allreduce_adam_p2p_hp with the guard.  A rank reduces only its own 1/R slice, so a norm phase sits between the two
 * barriers: every rank sums the squares of its reduced slice (per-CTA fp64 partials, added in CTA order by the last CTA), writes
 * that slice sum into every peer's flag area with a release, and every CTA adds the R slice sums in rank order — norm,
 * coefficient and skip decision are bit-identical on every rank.  A skipped step still sums the loss and runs the second barrier.
 *   peer_flags: >= DDFA_P2P_GUARD_FLAG_WORDS uint32 per rank (8-byte aligned), zero-initialised once;
 *   guard_state: ddfa_p2p_guard_state_bytes() LOCAL bytes, 16-byte aligned, zero-initialised once and kept between launches —
 *   two tickets, the per-CTA partials and the launch counter the barrier epochs come from (a skipped step does not advance
 *   step_count, so epochs cannot come from it).  The guarded and unguarded forms must not alternate on the same flag words.
 * gstate is written on every rank.  The step count is incremented by the kernel itself (one launch per step). */
#define DDFA_P2P_GUARD_FLAG_WORDS 96
size_t ddfa_p2p_guard_state_bytes(void);
int ddfa_allreduce_adam_p2p_guarded(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                                    int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                                    int64_t numel, int64_t loss_offset, float *loss_out, const float *hyper,
                                    const float *max_norm, float *gstate, int32_t *skipped, void *guard_state,
                                    void *stream);
/* Parameter groups over peer memory: ddfa_allreduce_adam_p2p_hp (ticket) and ddfa_allreduce_adam_p2p_guarded (guard_state) with
 * the ranges / groups of ddfa_adam_flat_groups in place of hyper (both LOCAL device buffers, the same values on every rank).
 * Each rank updates the intersection of its owned slice with the ranges; elements outside every range are neither read nor
 * written, on any rank.  Every updated element is bit-identical to ddfa_adam_flat_groups on the gradient summed in rank
 * order.  The guarded norm covers every element of every slice (the trainer zeroes gradients outside the ranges). */
int ddfa_allreduce_adam_p2p_groups(void *const *peer_params, const void *const *peer_grads, void *const *peer_flags,
                                   int32_t rank, int32_t world, float *exp_avg, float *exp_avg_sq, int32_t *step_count,
                                   int64_t numel, int64_t loss_offset, float *loss_out, uint32_t *ticket,
                                   const int64_t *ranges, int32_t num_ranges, const float *groups, int32_t num_groups,
                                   void *stream);
int ddfa_allreduce_adam_p2p_groups_guarded(void *const *peer_params, const void *const *peer_grads,
                                           void *const *peer_flags, int32_t rank, int32_t world, float *exp_avg,
                                           float *exp_avg_sq, int32_t *step_count, int64_t numel, int64_t loss_offset,
                                           float *loss_out, const int64_t *ranges, int32_t num_ranges,
                                           const float *groups, int32_t num_groups, const float *max_norm, float *gstate,
                                           int32_t *skipped, void *guard_state, void *stream);

/* ---------------------------------------------------------------------------------------
 * Gradient accumulation over micro-batches (Lightning's accumulate_grad_batches): elementwise over the elements
 * [begin, end) of two flat fp32 buffers, the accumulator `acc` and a micro-batch's gradients `grads`:
 *   DDFA_GRAD_ACC_SET   acc = grads    (the first micro-batch of a window)
 *   DDFA_GRAD_ACC_ADD   acc += grads   (the micro-batches after it)
 *   DDFA_GRAD_ACC_APPLY grads += acc   (the window's last micro-batch: the exchange and the update then read grads as always)
 * Both bounds multiples of 4, 0 <= begin <= end; acc and grads 16-byte aligned; nothing outside the range is read or written.
 * One launch (none for an empty range).  One fp32 add per element: bit-reproducible in both DDFA_TUNE_DETERMINISTIC modes.
 * ------------------------------------------------------------------------------------- */
#define DDFA_GRAD_ACC_SET 0
#define DDFA_GRAD_ACC_ADD 1
#define DDFA_GRAD_ACC_APPLY 2
int ddfa_grad_accumulate(float *acc, float *grads, int64_t begin, int64_t end, int32_t mode, void *stream);

/* ---------------------------------------------------------------------------------------
 * F2  processed Big-Vul files -> arena, on the device (csrc/csv_load.cu; SURVEY.md §8 row f2).  Replaces the host loaders
 * deepdfa_b200/bigvul_io.py restates: pd.read_csv of nodes.csv / edges.csv / nodes_feat_*.csv (written by DataFrame.to_csv,
 * DDFA/sastvd/scripts/dbize.py:104-105, dbize_absdf.py:44), the per-graph dgl.graph + add_self_loop of dbize_graphs.py:17-27,
 * the left merge of graphmogrifier.py:20-40 and the per-graph ndata of graphmogrifier.py:59-95.  Nothing here allocates:
 * every scratch buffer is a caller workspace sized by the matching *_workspace_bytes query.
 *
 * CSV dialect (pandas to_csv): ',' separates fields, '"' quotes them and "" escapes a quote inside; a row ends at a '\n' outside
 * quotes (an optional '\r' before it is dropped); blank lines are skipped.  Quote state is the parity of the quotes before a byte.
 *
 * ddfa_csv_index_count / ddfa_csv_index_rows: the row index of text[0, nbytes) (16-byte aligned; the caller appends a final
 *   '\n' when the file lacks one).  count writes info int64[2] = {rows, quote parity at the end (1: unterminated quote)};
 *   rows then sizes row_end int64[rows], which rows fills with the offset of each row's terminating '\n' (row 0: the header).
 *   Row r > 0 spans (row_end[r - 1], row_end[r]), blank lines before it skipped.  count: 2 launches, rows: 1.
 * ddfa_csv_fields: the data rows 1 .. rows-1 (output index r - 1), the columns at positions columns[0 .. num_columns)
 *   (ascending, at most DDFA_CSV_MAX_COLS) parsed to out[s] int64[rows - 1]: a signed decimal integer, optionally quoted,
 *   optionally followed by '.' and zeros.  Each row is read only up to its last requested column.  info int64[1 + 2 * num_columns]:
 *   [0] the first bad row, as the unsigned word (r - 1) << 8 | reason << 4 | slot (all ones: none; reason DDFA_CSV_ERR_NOT_INT
 *   or DDFA_CSV_ERR_NO_FIELD), then {min, max} of each column over the rows.  2 launches.
 * ddfa_row_sort: perm int32[n] = the row ids 0 .. n-1 stably sorted by (major[row], minor[row]) (minor NULL: by major alone),
 *   an LSD radix sort of 8-bit digits of key - key_min over key_bits bits (the host knows the range from ddfa_csv_fields).
 *   1 + 3 * (ceil(minor_bits / 8) + ceil(major_bits / 8)) launches.
 * ddfa_csv_graphs: the node rows sorted by graph_id (node_perm) form the graphs, in ascending graph_id; each graph's edges
 *   are the edge rows (sorted by graph_id: edge_perm) of its graph_id, in file row order.  Edge rows of other graph ids are not
 *   read.  info int64[DDFA_CSV_GRAPH_INFO_WORDS]: [0] G, [1] union edges (edge rows of the graphs + one self-loop per node),
 *   [2] the first bad graph as j << 8 | reason << 4 (all ones: none; DDFA_CSV_ERR_NO_EDGES, DDFA_CSV_ERR_NEGATIVE endpoint,
 *   DDFA_CSV_ERR_NODE_COUNT: max endpoint + 1 != node rows), for it [3] max endpoint + 1, [4] node rows, [5] graph_id.
 *   The workspace (ddfa_csv_graphs_workspace_bytes(node_rows)) carries the graph segments to ddfa_csv_union.  6-10 launches.
 * ddfa_csv_union (after ddfa_csv_graphs, with its workspace, num_graphs = info[0], when info[2] shows no error and
 *   info[1] < 2^31): the union COO src / dst int32[info[1]] = each graph's edge rows (src = innode, dst = outnode) offset by
 *   its first node, then its self-loops v -> v, graph after graph — what BG.batch of the add_self_loop'd graphs holds; arena
 *   node i = node row node_perm[i]; vuln int32[node_rows] = int32(float(vuln_col)) (attach_node_data's torch.Tensor(...).int());
 *   nodes_per_graph / edges_per_graph / graph_ids int64[G].  2 launches.
 * ddfa_csv_join: the left merge of one feature file on (graph_id, node_id): feat_perm sorts its rows by that pair
 *   (ddfa_row_sort); out[s][i] = values[s][the feature row of arena node i].  info int64[1]: the first arena node without a
 *   feature row (DDFA_CSV_ERR_NO_FEATURE) or with two (DDFA_CSV_ERR_DUPLICATE) as i << 8 | reason << 4; all ones: none.
 *   Workspace: the sorted keys, ddfa_csv_join_workspace_bytes(feature_rows).  1 memset + 2 launches.
 * Every entry runs on `stream` and reads no device word on the host.
 * ------------------------------------------------------------------------------------- */
#define DDFA_CSV_MAX_COLS 8
#define DDFA_CSV_GRAPH_INFO_WORDS 8
#define DDFA_CSV_ERR_NOT_INT 1
#define DDFA_CSV_ERR_NO_FIELD 2
#define DDFA_CSV_ERR_NO_EDGES 3
#define DDFA_CSV_ERR_NEGATIVE 4
#define DDFA_CSV_ERR_NODE_COUNT 5
#define DDFA_CSV_ERR_NO_FEATURE 6
#define DDFA_CSV_ERR_DUPLICATE 7
size_t ddfa_csv_index_workspace_bytes(int64_t nbytes);
int ddfa_csv_index_count(const uint8_t *text, int64_t nbytes, int64_t *info, void *workspace, size_t workspace_bytes, void *stream);
int ddfa_csv_index_rows(const uint8_t *text, int64_t nbytes, int64_t *row_end, void *workspace, size_t workspace_bytes, void *stream);
int ddfa_csv_fields(const uint8_t *text, const int64_t *row_end, int64_t rows, const int32_t *columns, int32_t num_columns,
                    int64_t *const *out, int64_t *info, void *stream);
size_t ddfa_row_sort_workspace_bytes(int32_t n);
int ddfa_row_sort(const int64_t *major, int64_t major_min, int32_t major_bits, const int64_t *minor, int64_t minor_min,
                  int32_t minor_bits, int32_t n, int32_t *perm, void *workspace, size_t workspace_bytes, void *stream);
size_t ddfa_csv_graphs_workspace_bytes(int32_t node_rows);
int ddfa_csv_graphs(const int64_t *node_gid, const int32_t *node_perm, int32_t node_rows, const int64_t *edge_gid,
                    const int32_t *edge_perm, int32_t edge_rows, const int64_t *innode, const int64_t *outnode, int64_t *info,
                    void *workspace, size_t workspace_bytes, void *stream);
int ddfa_csv_union(const int64_t *node_gid, const int32_t *node_perm, int32_t node_rows, const int64_t *vuln_col,
                   const int32_t *edge_perm, const int64_t *innode, const int64_t *outnode, int32_t num_graphs,
                   const void *workspace, size_t workspace_bytes, int32_t *src, int32_t *dst, int32_t *vuln,
                   int64_t *nodes_per_graph, int64_t *edges_per_graph, int64_t *graph_ids, void *stream);
size_t ddfa_csv_join_workspace_bytes(int32_t feature_rows);
int ddfa_csv_join(const int64_t *node_gid, const int64_t *node_nid, const int32_t *node_perm, int32_t node_rows,
                  const int64_t *feat_gid, const int64_t *feat_nid, const int32_t *feat_perm, int32_t feature_rows,
                  const int64_t *const *values, int32_t num_values, int64_t *const *out, int64_t *info, void *workspace,
                  size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Generic row-major fp32 GEMM on the SIMT engine (building block, exported for tests):
 *   C[M,N] = alpha * op(A) op(B) + beta * C,  op(X) = X or X^T per trans flag.
 * split_k > 1 accumulates partial products with atomics (requires beta == 1, C pre-initialised; rejected in deterministic mode).
 * ------------------------------------------------------------------------------------- */
int ddfa_sgemm(int trans_a, int trans_b, int32_t m, int32_t n, int32_t k, float alpha, const float *a,
               int32_t lda, const float *b, int32_t ldb, float beta, float *c, int32_t ldc,
               int32_t split_k, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DDFA_B200_H */
