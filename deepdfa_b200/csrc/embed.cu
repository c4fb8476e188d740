// K1 — embedding lookup + concat, forward and backward.
// Reference: 4x nn.Embedding(input_dim, hidden_dim) + torch.cat(dim=1) (ggnn.py:47-52,84-89) or a
// single nn.Embedding (ggnn.py:54,91-92).  Tables total 4*1002*32*4 B = 513 KB -> L2 resident;
// the op is bound by the index read (8 B/node/table) and the 4*D B/node output write.
#include <cuda_bf16.h>

#include "common.cuh"

namespace ddfa {

constexpr int kMaxTables = 8;
__device__ __forceinline__ uint32_t bf16x2_pack(float lo_half, float hi_half) {     // cvt.rn.bf16x2.f32: .x -> bits 0-15
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo_half, hi_half);
  return *reinterpret_cast<const uint32_t *>(&v);
}
struct EmbedPtrs {
  const int64_t *idx[kMaxTables];
  const float *table[kMaxTables];
  float *dtable[kMaxTables];
};

// one thread per 16-byte output chunk.  IMG (row width 128 only): the row also goes out as h_0's activation image (bf16 hi / lo,
// K-major SWIZZLE_128B tiles, include/ddfa_b200.h) — what a separate ddfa_act_to_image pass over x produced before.
template <bool IMG>
__global__ void __launch_bounds__(256) embed_concat_fwd_kernel(const EmbedPtrs p, int32_t K, int32_t V, int32_t H,
                                                               int32_t N, float *__restrict__ x, uint8_t *__restrict__ image,
                                                               int32_t *__restrict__ oob) {
  const int hq = H >> 2;           // chunks per table
  const int dq = K * hq;           // chunks per node row
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (int64_t)N * dq) return;
  const int32_t n = (int32_t)(t / dq);
  const int c = (int)(t - (int64_t)n * dq);
  const int k = c / hq, j = (c - k * hq) * 4;
  int64_t i = p.idx[k][n];
  if (i < 0 || i >= V) {
    if (oob && j == 0) atomicAdd(oob, 1);
    i = i < 0 ? 0 : V - 1;
  }
  const float4 v = ldg_nc_f4(p.table[k] + i * H + j);
  *reinterpret_cast<float4 *>(x + (int64_t)n * (K * H) + c * 4) = v;
  if constexpr (IMG) {
    const int col = c * 4, row = n & 127;
    const uint32_t h01 = bf16x2_pack(v.x, v.y), h23 = bf16x2_pack(v.z, v.w);
    const uint32_t l01 = bf16x2_pack(v.x - __uint_as_float(h01 << 16), v.y - __uint_as_float(h01 & 0xffff0000u));
    const uint32_t l23 = bf16x2_pack(v.z - __uint_as_float(h23 << 16), v.w - __uint_as_float(h23 & 0xffff0000u));
    uint8_t *tile = image + (size_t)(n >> 7) * 65536;
    const uint32_t sw = (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + (((((col & 63) >> 3) ^ (row & 7)) & 7) << 4) + (col & 7) * 2);
    *reinterpret_cast<uint2 *>(tile + (size_t)((0 * 2 + (col >> 6)) * 16384) + sw) = make_uint2(h01, h23);
    *reinterpret_cast<uint2 *>(tile + (size_t)((1 * 2 + (col >> 6)) * 16384) + sw) = make_uint2(l01, l23);
  }
}

// Backward: dtable[k][idx_k[n], :] += (dx + dx2)[n, kH:(k+1)H]   (dx2 optional).
// ~75 % of Big-Vul nodes carry index 0 ("not a definition", dbize_absdf.py:39) and a few % index 1
// (UNKNOWN), so rows 0 and 1 are privatised: each thread accumulates them in registers over its
// rows, the CTA reduces through shared memory and issues ONE RED per element per CTA; all other
// rows go straight to L2 with RED.ADD.F32.
__device__ __forceinline__ void red_add_f4(float *p, const float4 &v) {      // p 16-byte aligned (H % 4 == 0, tables 16-byte aligned)
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

constexpr int kEmbRows = 256;  // node rows per CTA
__global__ void __launch_bounds__(256) embed_concat_bwd_kernel(const EmbedPtrs p, int32_t K, int32_t V, int32_t H,
                                                               int32_t N, const float *__restrict__ dx,
                                                               const float *__restrict__ dx2) {
  extern __shared__ __align__(16) float red[];  // [ny][2][D]
  const int D = K * H;
  const int c = threadIdx.x;  // chunk inside the row (blockDim.x == D/4)
  const int hq = H >> 2;
  const int k = c / hq, j = (c - k * hq) * 4;
  const int64_t *idx = p.idx[k];
  float *dt = p.dtable[k];
  float4 hot[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  const int32_t row0 = blockIdx.x * kEmbRows;
  const int32_t row1 = min(N, row0 + kEmbRows);
  // four rows per iteration: their (independent) loads are in flight together — one row at a time was a chain of load latencies
  // (r03a launch list: 96 us for 157 MB at C1)
  constexpr int U = 4;
  for (int32_t nb = row0 + threadIdx.y; nb < row1; nb += U * blockDim.y) {
    float4 g[U];
    int64_t ii[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int32_t n = nb + u * blockDim.y;
      const bool ok = n < row1;
      g[u] = ok ? __ldg(reinterpret_cast<const float4 *>(dx + (int64_t)n * D + c * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (dx2 && ok) f4_add(g[u], __ldg(reinterpret_cast<const float4 *>(dx2 + (int64_t)n * D + c * 4)));
      ii[u] = ok ? idx[n] : -1;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (ii[u] == -1 && nb + u * (int32_t)blockDim.y >= row1) continue;
      int64_t i = ii[u];
      i = i < 0 ? 0 : (i >= V ? V - 1 : i);
      if (i == 0) f4_add(hot[0], g[u]);
      else if (i == 1) f4_add(hot[1], g[u]);
      else {
        red_add_f4(dt + i * H + j, g[u]);      // one 16-byte reduction instead of four (sm_90+: red.global.add.v4.f32)
      }
    }
  }
  *reinterpret_cast<float4 *>(&red[((size_t)threadIdx.y * 2 + 0) * D + c * 4]) = hot[0];
  *reinterpret_cast<float4 *>(&red[((size_t)threadIdx.y * 2 + 1) * D + c * 4]) = hot[1];
  __syncthreads();
  if (threadIdx.y < 2) {
    const int r = threadIdx.y;  // hot row 0 or 1
    if (r < V) {
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int y = 0; y < blockDim.y; ++y) f4_add(s, *reinterpret_cast<const float4 *>(&red[((size_t)y * 2 + r) * D + c * 4]));
      red_add_f4(dt + (int64_t)r * H + j, s);
    }
  }
}

// ---- deterministic backward (DDFA_TUNE_DETERMINISTIC = 1): a segmented sum over the nodes sorted by index ----------------
// Every table k sorts its node ids by index value with a stable counting sort: keys (k, i, c) count the nodes of chunk c (kDetChunk
// consecutive node ids) that carry index i in table k; their exclusive scan is where those nodes go, in node order inside the chunk.
// The sorted positions of table k are then cut into chunks of kDetChunk positions again: a team of lanes walks one chunk in order,
// adds a segment (one index) that lies inside the chunk straight into its gradient row, and leaves the partial sums of the segments
// that cross its ends in two slots; a last pass adds those slots in chunk order.  Index 0 (about 75 % of all nodes) is therefore
// summed by hundreds of teams in parallel, and every sum has one fixed order.
constexpr int kDetChunk = 256;

// one CTA (kDetChunk threads) per (chunk of node ids, table): count and in-chunk rank of each node's key
__global__ void __launch_bounds__(kDetChunk) embed_det_count_kernel(const EmbedPtrs p, int32_t V, int32_t N, int32_t nch,
                                                                     int32_t *__restrict__ cnt, int32_t *__restrict__ rank) {
  __shared__ int32_t s_i[kDetChunk];
  const int k = blockIdx.y, c = blockIdx.x, t = threadIdx.x;
  const int32_t n = c * kDetChunk + t;
  int32_t i = -1;
  if (n < N) {
    const int64_t v = p.idx[k][n];
    i = (int32_t)(v < 0 ? 0 : (v >= V ? V - 1 : v));
  }
  s_i[t] = i;
  __syncthreads();
  if (n >= N) return;
  int32_t r = 0;
  bool last = true;
  for (int j = 0; j < kDetChunk; ++j) {
    const bool same = s_i[j] == i;
    r += same && j < t;
    last = last && !(same && j > t);
  }
  rank[(int64_t)k * N + n] = r;
  if (last) cnt[1 + ((int64_t)k * V + i) * nch + c] = r + 1;   // a[0] = 0, counts from a[1] (scan_counts' layout)
}

// after the scan: cnt[key] = sorted position of the key's first node; node n goes to cnt[key] + its rank
__global__ void __launch_bounds__(256) embed_det_scatter_kernel(const EmbedPtrs p, int32_t V, int32_t N, int32_t nch,
                                                                 const int32_t *__restrict__ base, const int32_t *__restrict__ rank,
                                                                 int32_t *__restrict__ perm, int32_t *__restrict__ sidx) {
  const int k = blockIdx.y;
  const int32_t n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  const int64_t v = p.idx[k][n];
  const int32_t i = (int32_t)(v < 0 ? 0 : (v >= V ? V - 1 : v));
  const int32_t pos = base[((int64_t)k * V + i) * nch + n / kDetChunk] + rank[(int64_t)k * N + n];   // in [k N, (k + 1) N)
  perm[pos] = n;
  sidx[pos] = i;
}

// a team of TL lanes per chunk of sorted positions; lane tl owns the float4 columns tl + TL * w (w < COLS) of the table row (H / 4 of them)
template <int COLS>
__device__ __forceinline__ void team_add(float *row, const float4 (&acc)[COLS], int tl, int TL, int hq) {
#pragma unroll
  for (int w = 0; w < COLS; ++w) {
    const int q = tl + w * TL;
    if (q < hq) {
      float4 d = *reinterpret_cast<float4 *>(row + 4 * q);
      f4_add(d, acc[w]);
      *reinterpret_cast<float4 *>(row + 4 * q) = d;
    }
  }
}

template <int COLS>
__global__ void __launch_bounds__(256) embed_det_walk_kernel(const EmbedPtrs p, int32_t K, int32_t H, int32_t N, int32_t nch, int TL,
                                                              const float *__restrict__ dx, const float *__restrict__ dx2,
                                                              const int32_t *__restrict__ perm, const int32_t *__restrict__ sidx,
                                                              float *__restrict__ part) {
  const int k = blockIdx.y, hq = H >> 2, D = K * H;
  const int tl = threadIdx.x % TL;
  const int32_t c = (int32_t)((blockIdx.x * blockDim.x + threadIdx.x) / TL);
  if (c >= nch) return;
  const int32_t p0 = c * kDetChunk, p1 = min(N, p0 + kDetChunk);
  const int32_t *pm = perm + (int64_t)k * N, *si = sidx + (int64_t)k * N;
  float *dt = p.dtable[k];
  float *slot = part + ((int64_t)k * nch + c) * 2 * H;      // [head | tail] partial rows of this chunk
  float4 acc[COLS];
#pragma unroll
  for (int w = 0; w < COLS; ++w) acc[w] = make_float4(0.f, 0.f, 0.f, 0.f);
  int32_t cur = si[p0];
  bool head = true;                                         // the segment being summed contains p0
  const bool head_open = p0 > 0 && si[p0 - 1] == cur;       // ... and began in an earlier chunk
  auto flush = [&](bool open_end) {
    if ((head && head_open) || open_end) {
      float *dst = slot + (head ? 0 : H);
#pragma unroll
      for (int w = 0; w < COLS; ++w)
        if (tl + w * TL < hq) *reinterpret_cast<float4 *>(dst + 4 * (tl + w * TL)) = acc[w];
    } else {
      team_add<COLS>(dt + (int64_t)cur * H, acc, tl, TL, hq);     // the whole segment is in this chunk: its only writer
    }
#pragma unroll
    for (int w = 0; w < COLS; ++w) acc[w] = make_float4(0.f, 0.f, 0.f, 0.f);
  };
  constexpr int U = 8;      // positions in flight per lane
  for (int32_t pb = p0; pb < p1; pb += U) {
    int32_t nn[U], ii[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      nn[u] = pb + u < p1 ? pm[pb + u] : -1;
      ii[u] = pb + u < p1 ? si[pb + u] : -1;
    }
    float4 g[U][COLS];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int w = 0; w < COLS; ++w) {
        const int q = tl + w * TL;
        g[u][w] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (nn[u] >= 0 && q < hq) {
          const int64_t off = (int64_t)nn[u] * D + k * H + 4 * q;
          g[u][w] = __ldg(reinterpret_cast<const float4 *>(dx + off));
          if (dx2) f4_add(g[u][w], __ldg(reinterpret_cast<const float4 *>(dx2 + off)));
        }
      }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (nn[u] >= 0) {
        if (ii[u] != cur) {
          flush(false);
          cur = ii[u];
          head = false;
        }
#pragma unroll
        for (int w = 0; w < COLS; ++w) f4_add(acc[w], g[u][w]);
      }
    }
  }
  flush(p1 < N && si[p1] == cur);
}

// one team per (table, index) whose sorted segment crosses a chunk end: its chunk partials, added in chunk order
template <int COLS>
__global__ void __launch_bounds__(256) embed_det_combine_kernel(const EmbedPtrs p, int32_t K, int32_t V, int32_t H, int32_t N,
                                                                 int32_t nch, int TL, const int32_t *__restrict__ base,
                                                                 const float *__restrict__ part) {
  const int hq = H >> 2;
  const int tl = threadIdx.x % TL;
  const int64_t key = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / TL;      // k * V + i
  if (key >= (int64_t)K * V) return;
  const int k = (int)(key / V);
  const int32_t s = base[key * nch] - k * N, e = base[(key + 1) * nch] - k * N;   // base[K V nch] = K N (the scan's total)
  if (e - s < 2) return;
  const int32_t ca = s / kDetChunk, cb = (e - 1) / kDetChunk;
  if (ca == cb) return;
  const float *pk = part + (int64_t)k * nch * 2 * H;
  const int first = (s == ca * kDetChunk) ? 0 : 1;          // the segment is chunk ca's head only if it starts at ca's first position
  float4 acc[COLS];
#pragma unroll
  for (int w = 0; w < COLS; ++w) {
    const int q = tl + w * TL;
    acc[w] = q < hq ? *reinterpret_cast<const float4 *>(pk + ((int64_t)ca * 2 + first) * H + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  // chunks ca+1 .. cb go to kLanes interleaved accumulators (chunk c to accumulator (c - ca - 1) % kLanes), which are then added
  // in a fixed tree: the same order on every run, and kLanes independent load-add chains for index 0's hundreds of chunks
  constexpr int kLanes = 8;
  float4 part_acc[kLanes][COLS];
#pragma unroll
  for (int j = 0; j < kLanes; ++j)
#pragma unroll
    for (int w = 0; w < COLS; ++w) part_acc[j][w] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int32_t c0 = ca + 1; c0 <= cb; c0 += kLanes)
#pragma unroll
    for (int j = 0; j < kLanes; ++j)
#pragma unroll
      for (int w = 0; w < COLS; ++w) {
        const int q = tl + w * TL;
        if (q < hq && c0 + j <= cb) f4_add(part_acc[j][w], *reinterpret_cast<const float4 *>(pk + (int64_t)(c0 + j) * 2 * H + 4 * q));
      }
#pragma unroll
  for (int s = kLanes / 2; s > 0; s >>= 1)
#pragma unroll
    for (int j = 0; j < s; ++j)
#pragma unroll
      for (int w = 0; w < COLS; ++w) f4_add(part_acc[j][w], part_acc[j + s][w]);
#pragma unroll
  for (int w = 0; w < COLS; ++w) f4_add(acc[w], part_acc[0][w]);
  team_add<COLS>(p.dtable[k] + (key - (int64_t)k * V) * H, acc, tl, TL, hq);
}

struct EmbedDetLayout {
  int32_t nch, nkeys, nsums;
  size_t off_cnt, off_sums, off_rank, off_perm, off_sidx, off_part, total;
};
static EmbedDetLayout embed_det_layout(int32_t K, int32_t V, int32_t H, int32_t N) {
  EmbedDetLayout l{};
  l.nch = (N + kDetChunk - 1) / kDetChunk;
  l.nkeys = K * V * l.nch;
  l.nsums = scan_block_sums_len(l.nkeys);
  auto up = [](size_t b) { return (b + 255) / 256 * 256; };
  l.off_cnt = 0;
  l.off_sums = up(l.off_cnt + sizeof(int32_t) * ((size_t)l.nkeys + 1));
  l.off_rank = up(l.off_sums + sizeof(int32_t) * (size_t)l.nsums);
  l.off_perm = up(l.off_rank + sizeof(int32_t) * (size_t)K * N);
  l.off_sidx = up(l.off_perm + sizeof(int32_t) * (size_t)K * N);
  l.off_part = up(l.off_sidx + sizeof(int32_t) * (size_t)K * N);
  l.total = up(l.off_part + sizeof(float) * (size_t)K * l.nch * 2 * H);
  return l;
}

}  // namespace ddfa

extern "C" {

static int embed_fwd_impl(const char *who, const int64_t *const *idx, const float *const *tables, int32_t K, int32_t V, int32_t H, int32_t N,
                          float *x, void *image, int32_t *oob_count, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(K >= 1 && K <= kMaxTables && V > 0 && H > 0 && H % 4 == 0 && N >= 0,
               "%s: unsupported shape K=%d V=%d H=%d N=%d (H%%4==0, K<=%d)", who, K, V, H, N, kMaxTables);
  DDFA_REQUIRE(image == nullptr || K * H == 128, "%s: the activation image exists for row width 128 only (K*H=%d)", who, K * H);
  if (N == 0) return DDFA_OK;
  DDFA_REQUIRE(idx && tables && x && aligned16(x) && aligned16(image), "%s: NULL or unaligned pointer", who);
  EmbedPtrs p{};
  for (int k = 0; k < K; ++k) {
    DDFA_REQUIRE(idx[k] && tables[k] && aligned16(tables[k]), "%s: table %d pointer NULL or unaligned", who, k);
    p.idx[k] = idx[k];
    p.table[k] = tables[k];
  }
  const int64_t tot = (int64_t)N * K * (H / 4);
  const unsigned grid = (unsigned)((tot + 255) / 256);
  if (image) embed_concat_fwd_kernel<true><<<grid, 256, 0, as_stream(stream_)>>>(p, K, V, H, N, x, static_cast<uint8_t *>(image), oob_count);
  else embed_concat_fwd_kernel<false><<<grid, 256, 0, as_stream(stream_)>>>(p, K, V, H, N, x, nullptr, oob_count);
  DDFA_CHECK_LAUNCH("embed_concat_fwd_kernel");
  return DDFA_OK;
}

int ddfa_embed_concat_fwd(const int64_t *const *idx, const float *const *tables, int32_t K, int32_t V, int32_t H,
                          int32_t N, float *x, int32_t *oob_count, void *stream_) {
  return embed_fwd_impl("ddfa_embed_concat_fwd", idx, tables, K, V, H, N, x, nullptr, oob_count, stream_);
}

int ddfa_embed_concat_fwd_image(const int64_t *const *idx, const float *const *tables, int32_t K, int32_t V, int32_t H,
                                int32_t N, float *x, void *image, int32_t *oob_count, void *stream_) {
  DDFA_REQUIRE(image != nullptr, "ddfa_embed_concat_fwd_image: NULL image");
  return embed_fwd_impl("ddfa_embed_concat_fwd_image", idx, tables, K, V, H, N, x, image, oob_count, stream_);
}

size_t ddfa_embed_concat_bwd_workspace_bytes(int32_t K, int32_t V, int32_t H, int32_t N) {
  if (K < 1 || V < 1 || H < 1 || N < 0) return 0;
  return ddfa::embed_det_layout(K, V, H, N).total;
}

static int embed_bwd_impl(const char *who, const int64_t *const *idx, const float *dx, const float *dx2, int32_t K, int32_t V, int32_t H,
                          int32_t N, float *const *dtables, void *workspace, size_t workspace_bytes, bool has_ws, void *stream_) {
  using namespace ddfa;
  DDFA_REQUIRE(K >= 1 && K <= kMaxTables && V > 0 && H > 0 && H % 4 == 0 && N >= 0 && K * H <= 512,
               "%s: unsupported shape K=%d V=%d H=%d N=%d", who, K, V, H, N);
  DDFA_REQUIRE(has_ws || !deterministic(),
               "ddfa_embed_concat_bwd has no deterministic form (DDFA_TUNE_DETERMINISTIC = 1): use ddfa_embed_concat_bwd_ws");
  if (N == 0) return DDFA_OK;
  if (deterministic()) {
    const EmbedDetLayout l = embed_det_layout(K, V, H, N);
    DDFA_REQUIRE((int64_t)K * V * l.nch < ((int64_t)1 << 31) - 1, "%s: K * V * ceil(N / %d) exceeds int32", who, kDetChunk);
    if (workspace == nullptr || workspace_bytes < l.total) {
      set_error("%s: workspace too small (%zu < %zu)", who, workspace_bytes, l.total);
      return DDFA_ERR_WORKSPACE;
    }
    DDFA_REQUIRE(idx && dx && dtables && aligned16(dx) && aligned16(dx2) && aligned16(workspace), "%s: NULL or unaligned pointer", who);
    EmbedPtrs p{};
    for (int k = 0; k < K; ++k) {
      DDFA_REQUIRE(idx[k] && dtables[k] && aligned16(dtables[k]), "%s: table %d pointer NULL or unaligned", who, k);
      p.idx[k] = idx[k];
      p.dtable[k] = dtables[k];
    }
    cudaStream_t stream = as_stream(stream_);
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws + l.off_cnt), *sums = reinterpret_cast<int32_t *>(ws + l.off_sums);
    int32_t *rank = reinterpret_cast<int32_t *>(ws + l.off_rank), *perm = reinterpret_cast<int32_t *>(ws + l.off_perm);
    int32_t *sidx = reinterpret_cast<int32_t *>(ws + l.off_sidx);
    float *part = reinterpret_cast<float *>(ws + l.off_part);
    DDFA_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * ((size_t)l.nkeys + 1), stream));
    embed_det_count_kernel<<<dim3(l.nch, K), kDetChunk, 0, stream>>>(p, V, N, l.nch, cnt, rank);
    DDFA_CHECK_LAUNCH("embed_det_count_kernel");
    const int rc = scan_counts(cnt, nullptr, l.nkeys, sums, nullptr, stream);
    if (rc != DDFA_OK) return rc;
    embed_det_scatter_kernel<<<dim3((N + 255) / 256, K), 256, 0, stream>>>(p, V, N, l.nch, cnt, rank, perm, sidx);
    DDFA_CHECK_LAUNCH("embed_det_scatter_kernel");
    const int hq = H / 4;
    int TL = 1;
    while (TL < hq && TL < 32) TL *= 2;
    const unsigned walk_blocks = (unsigned)(((int64_t)l.nch * TL + 255) / 256), comb_blocks = (unsigned)(((int64_t)K * V * TL + 255) / 256);
    if (hq <= 32) {
      embed_det_walk_kernel<1><<<dim3(walk_blocks, K), 256, 0, stream>>>(p, K, H, N, l.nch, TL, dx, dx2, perm, sidx, part);
      DDFA_CHECK_LAUNCH("embed_det_walk_kernel");
      embed_det_combine_kernel<1><<<comb_blocks, 256, 0, stream>>>(p, K, V, H, N, l.nch, TL, cnt, part);
    } else {
      embed_det_walk_kernel<4><<<dim3(walk_blocks, K), 256, 0, stream>>>(p, K, H, N, l.nch, TL, dx, dx2, perm, sidx, part);
      DDFA_CHECK_LAUNCH("embed_det_walk_kernel");
      embed_det_combine_kernel<4><<<comb_blocks, 256, 0, stream>>>(p, K, V, H, N, l.nch, TL, cnt, part);
    }
    DDFA_CHECK_LAUNCH("embed_det_combine_kernel");
    return DDFA_OK;
  }
  DDFA_REQUIRE(idx && dx && dtables && aligned16(dx) && aligned16(dx2), "%s: NULL or unaligned pointer", who);
  for (int k = 0; k < K; ++k) DDFA_REQUIRE(aligned16(dtables[k]), "%s: gradient table %d must be 16-byte aligned", who, k);
  EmbedPtrs p{};
  for (int k = 0; k < K; ++k) {
    DDFA_REQUIRE(idx[k] && dtables[k], "%s: table %d pointer NULL", who, k);
    p.idx[k] = idx[k];
    p.dtable[k] = dtables[k];
  }
  const int D = K * H;
  dim3 block(D / 4, (256 / (D / 4)) > 2 ? 256 / (D / 4) : 2);
  const size_t smem = sizeof(float) * block.y * 2 * D;
  embed_concat_bwd_kernel<<<(N + kEmbRows - 1) / kEmbRows, block, smem, as_stream(stream_)>>>(p, K, V, H, N, dx, dx2);
  DDFA_CHECK_LAUNCH("embed_concat_bwd_kernel");
  return DDFA_OK;
}

int ddfa_embed_concat_bwd(const int64_t *const *idx, const float *dx, const float *dx2, int32_t K, int32_t V, int32_t H,
                          int32_t N, float *const *dtables, void *stream_) {
  return embed_bwd_impl("ddfa_embed_concat_bwd", idx, dx, dx2, K, V, H, N, dtables, nullptr, 0, false, stream_);
}

int ddfa_embed_concat_bwd_ws(const int64_t *const *idx, const float *dx, const float *dx2, int32_t K, int32_t V, int32_t H,
                             int32_t N, float *const *dtables, void *workspace, size_t workspace_bytes, void *stream_) {
  return embed_bwd_impl("ddfa_embed_concat_bwd_ws", idx, dx, dx2, K, V, H, N, dtables, workspace, workspace_bytes, true, stream_);
}

}  // extern "C"
