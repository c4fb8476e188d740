// The reference's processed Big-Vul CSV files (nodes.csv, edges.csv, nodes_feat_*.csv, written by DataFrame.to_csv) parsed,
// grouped and joined on the device into the arena's union COO and node data (layout and rules in include/ddfa_b200.h, F2).
//
//   row index:  fixed chunks of kChunk bytes count their quotes and their newlines under both parities; a one-CTA scan gives
//               the quote parity at each chunk's start and the row ends before it; a scatter writes the byte offset of every
//               newline at even parity (a "" escape toggles twice) that does not end a blank line.
//   fields:     one thread per row walks its bytes up to the last requested column and parses those columns to int64.
//   sort:       LSD radix sort (8-bit digits) of the row ids, the key gathered per row from its int64 column; stable, so a
//               minor column's passes followed by a major column's give the lexicographic order.
//   graphs:     segments of the node rows sorted by graph_id; per graph (one warp) its edge segment by binary search, the
//               segmented maximum / minimum of the endpoints, the node-count check; then the union COO.
//   join:       per arena node a binary search of (graph_id, node_id) in a feature file's sorted keys.
// Errors go to device words (atomicMin of row-or-graph << 8 | reason << 4 | column slot), read by the host after the call.
#include "common.cuh"

namespace ddfa {
namespace csv {

constexpr int kThreads = 256;
constexpr int kBytes = 16;                       // bytes per thread in the row index
constexpr int64_t kChunk = kThreads * kBytes;    // 4096 bytes per CTA
constexpr int kWarps = kThreads / 32;
constexpr int kBins = 256;
constexpr int kItems = 16;
constexpr int kTile = kThreads * kItems;         // 4096 row ids per sort tile
constexpr int kWarpSpan = 32 * kItems;

inline size_t align16(size_t b) { return (b + 15) & ~size_t(15); }
inline int64_t num_chunks(int64_t n) { return (n + kChunk - 1) / kChunk; }
inline int64_t num_tiles(int64_t n) { return (n + kTile - 1) / kTile; }

// ---- row index ---------------------------------------------------------------------------------------------------------
// a newline at even parity ends a blank line (skipped, as read_csv skips it) when the line before it ended right there
__device__ __forceinline__ bool blank_line_end(const uint8_t *t, int64_t i) {
  if (i == 0) return true;
  const uint8_t p = t[i - 1];
  if (p == '\n') return true;
  return p == '\r' && (i == 1 || t[i - 2] == '\n');
}

__device__ __forceinline__ void load_bytes(const uint8_t *t, int64_t n, int64_t i0, uint8_t (&b)[kBytes]) {
  if (i0 + kBytes <= n) {
    const uint4 v = *reinterpret_cast<const uint4 *>(t + i0);
    const uint8_t *p = reinterpret_cast<const uint8_t *>(&v);
#pragma unroll
    for (int j = 0; j < kBytes; ++j) b[j] = p[j];
  } else {
#pragma unroll
    for (int j = 0; j < kBytes; ++j) b[j] = i0 + j < n ? t[i0 + j] : 0;
  }
}

// exclusive XOR prefix of one bit over the CTA's threads, and the CTA's total
__device__ __forceinline__ int block_xor_excl(int q, int &total) {
  __shared__ int wpar[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, q);
  if (lane == 0) wpar[warp] = __popc(m) & 1;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    before ^= w < warp ? wpar[w] : 0;
    total ^= wpar[w];
  }
  __syncthreads();
  return before ^ (__popc(m & ((1u << lane) - 1u)) & 1);
}

// exclusive sum over the CTA's threads, and the CTA's total
__device__ __forceinline__ int64_t block_sum_excl(int64_t v, int64_t &total) {
  __shared__ int64_t ws[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[warp] = x;
  __syncthreads();
  int64_t before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    before += w < warp ? ws[w] : 0;
    total += ws[w];
  }
  __syncthreads();
  return before + x - v;
}

// per chunk: quote parity, and the row ends it holds if it starts at even (cnt0) or odd (cnt1) parity
__global__ void __launch_bounds__(kThreads) index_count_kernel(const uint8_t *__restrict__ t, int64_t n, int32_t *__restrict__ qpar,
                                                               int32_t *__restrict__ cnt0, int32_t *__restrict__ cnt1) {
  const int64_t i0 = blockIdx.x * kChunk + threadIdx.x * (int64_t)kBytes;
  uint8_t b[kBytes];
  load_bytes(t, n, i0, b);
  int q = 0, e0 = 0, e1 = 0;      // e0: row ends at even parity from this thread's start, e1: at odd
#pragma unroll
  for (int j = 0; j < kBytes; ++j) {
    if (b[j] == '"') q ^= 1;
    else if (b[j] == '\n' && i0 + j < n && !blank_line_end(t, i0 + j)) {
      e0 += q == 0;
      e1 += q != 0;
    }
  }
  int qtot;
  const int pt = block_xor_excl(q, qtot);
  int64_t c0, c1;
  block_sum_excl(pt ? e1 : e0, c0);
  block_sum_excl(pt ? e0 : e1, c1);
  if (threadIdx.x == 0) {
    qpar[blockIdx.x] = qtot;
    cnt0[blockIdx.x] = (int32_t)c0;
    cnt1[blockIdx.x] = (int32_t)c1;
  }
}

// one CTA, chunks in order: qpar -> the parity at each chunk's start (in place), off = row ends before each chunk;
// info[0] = rows, info[1] = the parity at the end of the text (1: a quote is never closed)
__global__ void __launch_bounds__(kThreads) index_scan_kernel(int32_t *__restrict__ qpar, const int32_t *__restrict__ cnt0,
                                                              const int32_t *__restrict__ cnt1, int64_t chunks, int64_t *__restrict__ off,
                                                              int64_t *__restrict__ info) {
  int par = 0;
  int64_t carry = 0;
  for (int64_t c0 = 0; c0 < chunks; c0 += kThreads) {
    const int64_t c = c0 + threadIdx.x;
    const int q = c < chunks ? qpar[c] : 0;
    int qt;
    const int pin = par ^ block_xor_excl(q, qt);
    const int64_t v = c < chunks ? (pin ? cnt1[c] : cnt0[c]) : 0;
    int64_t tot;
    const int64_t ex = block_sum_excl(v, tot);
    if (c < chunks) {
      qpar[c] = pin;
      off[c] = carry + ex;
    }
    par ^= qt;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    info[0] = carry;
    info[1] = par;
  }
}

__global__ void __launch_bounds__(kThreads) index_scatter_kernel(const uint8_t *__restrict__ t, int64_t n, const int32_t *__restrict__ pin,
                                                                 const int64_t *__restrict__ off, int64_t *__restrict__ row_end) {
  const int64_t i0 = blockIdx.x * kChunk + threadIdx.x * (int64_t)kBytes;
  uint8_t b[kBytes];
  load_bytes(t, n, i0, b);
  int q = 0;
#pragma unroll
  for (int j = 0; j < kBytes; ++j) q ^= b[j] == '"';
  int qt;
  int p = pin[blockIdx.x] ^ block_xor_excl(q, qt);
  uint32_t ends = 0;
#pragma unroll
  for (int j = 0; j < kBytes; ++j) {
    if (b[j] == '"') p ^= 1;
    else if (b[j] == '\n' && p == 0 && i0 + j < n && !blank_line_end(t, i0 + j)) ends |= 1u << j;
  }
  int64_t tot;
  int64_t pos = off[blockIdx.x] + block_sum_excl(__popc(ends), tot);
#pragma unroll
  for (int j = 0; j < kBytes; ++j)
    if (ends >> j & 1u) row_end[pos++] = i0 + j;
}

// ---- fields ----------------------------------------------------------------------------------------------------------
// a signed decimal integer, optionally "quoted", optionally followed by '.' and zeros (an integral float written by to_csv)
__device__ bool parse_i64(const uint8_t *t, int64_t a, int64_t b, int64_t &out) {
  if (b - a >= 2 && t[a] == '"' && t[b - 1] == '"') {
    ++a;
    --b;
  }
  bool neg = false;
  if (a < b && (t[a] == '-' || t[a] == '+')) {
    neg = t[a] == '-';
    ++a;
  }
  const uint64_t limit = neg ? (1ull << 63) : (1ull << 63) - 1;
  uint64_t acc = 0;
  int digits = 0;
  for (; a < b && t[a] >= '0' && t[a] <= '9'; ++a, ++digits) {
    const uint64_t d = t[a] - '0';
    if (acc > (limit - d) / 10) return false;
    acc = acc * 10 + d;
  }
  if (digits == 0) return false;
  if (a < b && t[a] == '.')
    for (++a; a < b && t[a] == '0'; ++a) {
    }
  if (a != b) return false;
  out = neg ? (int64_t)(0ull - acc) : (int64_t)acc;
  return true;
}

struct FieldArgs {
  int32_t col[DDFA_CSV_MAX_COLS];      // column positions, ascending
  int64_t *out[DDFA_CSV_MAX_COLS];
};

__global__ void fields_init_kernel(int64_t *info, int ncol) {
  const int i = threadIdx.x;
  if (i == 0) info[0] = -1;                                    // all bits set: no error (atomicMin as unsigned)
  if (i < ncol) {
    info[1 + 2 * i] = INT64_MAX;
    info[2 + 2 * i] = INT64_MIN;
  }
}

// thread per data row r (file row r + 1: row 0 is the header)
__global__ void __launch_bounds__(kThreads) fields_kernel(const uint8_t *__restrict__ t, const int64_t *__restrict__ row_end, int64_t rows,
                                                          FieldArgs a, int ncol, int64_t *__restrict__ info) {
  const int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  int64_t lo[DDFA_CSV_MAX_COLS], hi[DDFA_CSV_MAX_COLS];
#pragma unroll
  for (int s = 0; s < DDFA_CSV_MAX_COLS; ++s) {
    lo[s] = INT64_MAX;
    hi[s] = INT64_MIN;
  }
  if (r < rows) {
    int64_t p = row_end[r] + 1, e = row_end[r + 1];
    while (p < e && (t[p] == '\n' || t[p] == '\r')) ++p;      // the blank lines before the row
    if (e > p && t[e - 1] == '\r') --e;                        // \r\n
    int slot = 0, f = 0;
    int64_t fs = p;
    bool inq = false;
    unsigned long long bad = 0;
    for (;; ++p) {
      const bool at_end = p == e;
      const uint8_t ch = at_end ? 0 : t[p];
      if (ch == '"') {
        inq = !inq;
        continue;
      }
      if (at_end || (ch == ',' && !inq)) {
        if (f == a.col[slot]) {
          int64_t v;
          if (!parse_i64(t, fs, p, v)) {
            bad = (unsigned long long)r << 8 | DDFA_CSV_ERR_NOT_INT << 4 | slot;
            break;
          }
          a.out[slot][r] = v;
          lo[slot] = v;
          hi[slot] = v;
          if (++slot == ncol) break;
        }
        if (at_end) {
          bad = (unsigned long long)r << 8 | DDFA_CSV_ERR_NO_FIELD << 4 | slot;
          break;
        }
        ++f;
        fs = p + 1;
      }
    }
    if (bad) atomicMin(reinterpret_cast<unsigned long long *>(info), bad);
  }
  for (int s = 0; s < ncol; ++s) {
    int64_t l = lo[s], h = hi[s];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      l = min(l, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)l, o));
      h = max(h, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)h, o));
    }
    if ((threadIdx.x & 31) == 0 && l <= h) {
      atomicMin(reinterpret_cast<long long *>(info + 1 + 2 * s), (long long)l);
      atomicMax(reinterpret_cast<long long *>(info + 2 + 2 * s), (long long)h);
    }
  }
}

// ---- LSD radix sort of row ids by a gathered int64 key ------------------------------------------------------------------
__device__ __forceinline__ int digit_of(const int64_t *key, int64_t kmin, int shift, int32_t row) {
  return (int)((((uint64_t)key[row] - (uint64_t)kmin) >> shift) & (kBins - 1));
}

__global__ void iota_kernel(int32_t *p, int32_t n) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i < n) p[i] = i;
}

__global__ void __launch_bounds__(kThreads) sort_count_kernel(const int32_t *__restrict__ in, int32_t n, const int64_t *__restrict__ key,
                                                              int64_t kmin, int shift, int32_t tiles, int32_t *__restrict__ counts) {
  __shared__ int32_t h[kBins];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = blockIdx.x * (int64_t)kTile;
#pragma unroll 4
  for (int k = 0; k < kItems; ++k) {
    const int64_t i = base + k * kThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[digit_of(key, kmin, shift, in[i])], 1);
  }
  __syncthreads();
  counts[threadIdx.x * (int64_t)tiles + blockIdx.x] = h[threadIdx.x];
}

// CTA per digit: its tile counts -> exclusive prefix across tiles (in place), its total -> row_total
__global__ void __launch_bounds__(kThreads) sort_scan_kernel(int32_t *__restrict__ counts, int32_t tiles, int32_t *__restrict__ row_total) {
  int32_t *row = counts + blockIdx.x * (int64_t)tiles;
  int64_t carry = 0;
  for (int32_t c0 = 0; c0 < tiles; c0 += kThreads) {
    const int32_t i = c0 + threadIdx.x;
    const int64_t v = i < tiles ? row[i] : 0;
    int64_t tot;
    const int64_t ex = block_sum_excl(v, tot);
    if (i < tiles) row[i] = (int32_t)(carry + ex);
    carry += tot;
  }
  if (threadIdx.x == 0) row_total[blockIdx.x] = (int32_t)carry;
}

// stable scatter: warps own consecutive spans of the tile, rounds in order, lanes in order (__match_any_sync ranks)
__global__ void __launch_bounds__(kThreads) sort_scatter_kernel(const int32_t *__restrict__ in, int32_t n, const int64_t *__restrict__ key,
                                                                int64_t kmin, int shift, int32_t tiles, const int32_t *__restrict__ counts,
                                                                const int32_t *__restrict__ row_total, int32_t *__restrict__ out) {
  __shared__ int32_t start[kWarps][kBins];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  const int64_t base = blockIdx.x * (int64_t)kTile + warp * kWarpSpan;
  for (int j = threadIdx.x; j < kWarps * kBins; j += kThreads) (&start[0][0])[j] = 0;
  __syncthreads();
  int32_t v[kItems];
  int d[kItems];
#pragma unroll
  for (int it = 0; it < kItems; ++it) {
    const int64_t i = base + it * 32 + lane;
    const bool valid = i < n;
    v[it] = valid ? in[i] : 0;
    d[it] = valid ? digit_of(key, kmin, shift, v[it]) : kBins;
    const uint32_t peers = __match_any_sync(0xffffffffu, d[it]);
    if (valid && lane == __ffs(peers) - 1) start[warp][d[it]] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {
    const int b = threadIdx.x;
    const int64_t tot = row_total[b];
    int64_t all;
    int64_t run = block_sum_excl(tot, all) + counts[b * (int64_t)tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const int32_t c = start[w][b];
      start[w][b] = (int32_t)run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kItems; ++it) {
    const uint32_t peers = __match_any_sync(0xffffffffu, d[it]);
    if (d[it] < kBins) out[start[warp][d[it]] + __popc(peers & lt)] = v[it];
    __syncwarp();
    if (d[it] < kBins && lane == __ffs(peers) - 1) start[warp][d[it]] += __popc(peers);
    __syncwarp();
  }
}

struct SortWs {
  int32_t *tmp, *counts, *row_total;
};
inline size_t sort_layout(int32_t n, void *base, SortWs *w) {
  char *p = static_cast<char *>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) -> void * {
    void *q = p ? p + off : nullptr;
    off += align16(bytes);
    return q;
  };
  w->tmp = static_cast<int32_t *>(take(sizeof(int32_t) * (size_t)n));
  w->counts = static_cast<int32_t *>(take(sizeof(int32_t) * kBins * (size_t)num_tiles(n)));
  w->row_total = static_cast<int32_t *>(take(sizeof(int32_t) * kBins));
  return off;
}

// ---- graphs ----------------------------------------------------------------------------------------------------------
struct GraphWs {
  int32_t *gidx;      // [Rn + 1]: head flags of the sorted node rows, scanned in place -> graph index + 1 of each
  int32_t *sums0;     // block sums of the scans
  int32_t *node_off;  // [Rn + 1]: first sorted node row of each graph, then Rn
  int32_t *elo;       // [Rn]: first sorted edge row of each graph
  int32_t *eoff;      // [Rn + 1]: union edges of each graph (its edge rows + its self-loops), scanned in place -> offsets
  int32_t *sums1;
  int64_t *implied;   // [Rn]: max endpoint + 1 of each graph (for the error message)
};
inline size_t graph_layout(int32_t rn, void *base, GraphWs *w) {
  char *p = static_cast<char *>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) -> void * {
    void *q = p ? p + off : nullptr;
    off += align16(bytes);
    return q;
  };
  const size_t sl = rn > 0 ? (size_t)scan_block_sums_len(rn) : 1;
  w->gidx = static_cast<int32_t *>(take(sizeof(int32_t) * ((size_t)rn + 1)));
  w->sums0 = static_cast<int32_t *>(take(sizeof(int32_t) * sl));
  w->node_off = static_cast<int32_t *>(take(sizeof(int32_t) * ((size_t)rn + 1)));
  w->elo = static_cast<int32_t *>(take(sizeof(int32_t) * (size_t)rn));
  w->eoff = static_cast<int32_t *>(take(sizeof(int32_t) * ((size_t)rn + 1)));
  w->sums1 = static_cast<int32_t *>(take(sizeof(int32_t) * sl));
  w->implied = static_cast<int64_t *>(take(sizeof(int64_t) * (size_t)rn));
  return off;
}

__device__ __forceinline__ bool is_head(const int64_t *gid, const int32_t *perm, int32_t i) {
  return i == 0 || gid[perm[i]] != gid[perm[i - 1]];
}

__global__ void head_kernel(const int64_t *__restrict__ gid, const int32_t *__restrict__ perm, int32_t rn, int32_t *__restrict__ gidx) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i == 0) gidx[0] = 0;
  if (i < rn) gidx[i + 1] = is_head(gid, perm, i);
}

__global__ void node_off_kernel(const int64_t *__restrict__ gid, const int32_t *__restrict__ perm, int32_t rn, const int32_t *__restrict__ gidx,
                                int32_t *__restrict__ node_off) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= rn) return;
  if (is_head(gid, perm, i)) node_off[gidx[i + 1] - 1] = i;
  if (i == rn - 1) node_off[gidx[rn]] = rn;
}

// first sorted position in [0, n) whose key is >= g (upper = false) or > g (upper = true)
__device__ __forceinline__ int32_t bound(const int64_t *key, const int32_t *perm, int32_t n, int64_t g, bool upper) {
  int32_t lo = 0, hi = n;
  while (lo < hi) {
    const int32_t mid = lo + (hi - lo) / 2;
    const int64_t k = key[perm[mid]];
    if (upper ? k <= g : k < g) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// warp per graph (grid-stride): its edge segment, the endpoint range, the checks, its union edge count
__global__ void __launch_bounds__(kThreads) graph_kernel(const int64_t *__restrict__ node_gid, const int32_t *__restrict__ node_perm,
                                                         int32_t rn, const int64_t *__restrict__ edge_gid, const int32_t *__restrict__ edge_perm,
                                                         int32_t re, const int64_t *__restrict__ innode, const int64_t *__restrict__ outnode,
                                                         GraphWs w, int64_t *__restrict__ info) {
  const int lane = threadIdx.x & 31;
  const int32_t G = w.gidx[rn];
  for (int32_t j = (blockIdx.x * kThreads + threadIdx.x) >> 5; j < G; j += (gridDim.x * kThreads) >> 5) {
    const int32_t n0 = w.node_off[j], nn = w.node_off[j + 1] - n0;
    const int64_t g = node_gid[node_perm[n0]];
    int32_t lo = 0, hi = 0;
    if (lane == 0) {
      lo = bound(edge_gid, edge_perm, re, g, false);
      hi = bound(edge_gid, edge_perm, re, g, true);
    }
    lo = __shfl_sync(0xffffffffu, lo, 0);
    hi = __shfl_sync(0xffffffffu, hi, 0);
    int64_t mx = -1, mn = 0;
    for (int32_t k = lo + lane; k < hi; k += 32) {
      const int32_t r = edge_perm[k];
      const int64_t a = innode[r], b = outnode[r];
      mx = max(mx, max(a, b));
      mn = min(mn, min(a, b));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mx = max(mx, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)mx, o));
      mn = min(mn, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)mn, o));
    }
    if (lane == 0) {
      w.elo[j] = lo;
      w.implied[j] = mx + 1;
      const int64_t ue = (int64_t)(hi - lo) + nn;
      w.eoff[j + 1] = ue < INT32_MAX ? (int32_t)ue : INT32_MAX;
      atomicAdd(reinterpret_cast<unsigned long long *>(info + 1), (unsigned long long)ue);
      int reason = 0;
      if (hi == lo) reason = DDFA_CSV_ERR_NO_EDGES;
      else if (mn < 0) reason = DDFA_CSV_ERR_NEGATIVE;
      else if (mx + 1 != nn) reason = DDFA_CSV_ERR_NODE_COUNT;
      if (reason) atomicMin(reinterpret_cast<unsigned long long *>(info + 2), (unsigned long long)j << 8 | reason << 4);
    }
  }
}

// info[0] = G; for the first bad graph j (info[2]): its max endpoint + 1, node rows and graph_id for the message
__global__ void graph_info_kernel(const int64_t *node_gid, const int32_t *node_perm, GraphWs w, int32_t rn, int64_t *info) {
  info[0] = w.gidx[rn];
  w.eoff[0] = 0;
  const unsigned long long bad = (unsigned long long)info[2];
  if (bad != ~0ull) {
    const int32_t j = (int32_t)(bad >> 8);
    info[3] = w.implied[j];
    info[4] = w.node_off[j + 1] - w.node_off[j];
    info[5] = node_gid[node_perm[w.node_off[j]]];
  }
}

// warp per graph: its edge rows offset by its first node, then one self-loop per node; its sizes and id
__global__ void __launch_bounds__(kThreads) union_kernel(const int64_t *__restrict__ node_gid, const int32_t *__restrict__ node_perm,
                                                         const int32_t *__restrict__ edge_perm, const int64_t *__restrict__ innode,
                                                         const int64_t *__restrict__ outnode, GraphWs w, int32_t G, int32_t *__restrict__ src,
                                                         int32_t *__restrict__ dst, int64_t *__restrict__ nodes_per_graph,
                                                         int64_t *__restrict__ edges_per_graph, int64_t *__restrict__ graph_ids) {
  const int lane = threadIdx.x & 31;
  for (int32_t j = (blockIdx.x * kThreads + threadIdx.x) >> 5; j < G; j += (gridDim.x * kThreads) >> 5) {
    const int32_t n0 = w.node_off[j], nn = w.node_off[j + 1] - n0;
    const int32_t e0 = w.eoff[j], ne = w.eoff[j + 1] - e0, lo = w.elo[j], ke = ne - nn;
    for (int32_t k = lane; k < ke; k += 32) {
      const int32_t r = edge_perm[lo + k];
      src[e0 + k] = n0 + (int32_t)innode[r];
      dst[e0 + k] = n0 + (int32_t)outnode[r];
    }
    for (int32_t v = lane; v < nn; v += 32) src[e0 + ke + v] = dst[e0 + ke + v] = n0 + v;
    if (lane == 0) {
      nodes_per_graph[j] = nn;
      edges_per_graph[j] = ne;
      graph_ids[j] = node_gid[node_perm[n0]];
    }
  }
}

// _VULN as attach_node_data stores it: torch.Tensor(list).int(), i.e. through fp32
__global__ void vuln_kernel(const int64_t *__restrict__ vuln_col, const int32_t *__restrict__ node_perm, int32_t rn, int32_t *__restrict__ vuln) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i < rn) vuln[i] = (int32_t)__ll2float_rn((long long)vuln_col[node_perm[i]]);
}

// ---- join ------------------------------------------------------------------------------------------------------------
__global__ void join_keys_kernel(const int64_t *__restrict__ fg, const int64_t *__restrict__ fk, const int32_t *__restrict__ perm, int32_t rf,
                                 int64_t *__restrict__ sg, int64_t *__restrict__ sk) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i < rf) {
    sg[i] = fg[perm[i]];
    sk[i] = fk[perm[i]];
  }
}

struct JoinArgs {
  const int64_t *val[DDFA_CSV_MAX_COLS];
  int64_t *out[DDFA_CSV_MAX_COLS];
};

// thread per arena node i (node row node_perm[i]): lower bound of its key in the sorted feature keys
__global__ void __launch_bounds__(kThreads) join_kernel(const int64_t *__restrict__ node_gid, const int64_t *__restrict__ node_nid,
                                                        const int32_t *__restrict__ node_perm, int32_t rn, const int64_t *__restrict__ sg,
                                                        const int64_t *__restrict__ sk, const int32_t *__restrict__ feat_perm, int32_t rf,
                                                        JoinArgs a, int ncol, int64_t *__restrict__ info) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= rn) return;
  const int32_t r = node_perm[i];
  const int64_t g = node_gid[r], k = node_nid[r];
  int32_t lo = 0, hi = rf;
  while (lo < hi) {
    const int32_t mid = lo + (hi - lo) / 2;
    const int64_t mg = sg[mid];
    if (mg < g || (mg == g && sk[mid] < k)) lo = mid + 1;
    else hi = mid;
  }
  int reason = 0;
  if (lo == rf || sg[lo] != g || sk[lo] != k) reason = DDFA_CSV_ERR_NO_FEATURE;
  else if (lo + 1 < rf && sg[lo + 1] == g && sk[lo + 1] == k) reason = DDFA_CSV_ERR_DUPLICATE;
  if (reason) {
    atomicMin(reinterpret_cast<unsigned long long *>(info), (unsigned long long)i << 8 | reason << 4);
    return;
  }
  const int32_t fr = feat_perm[lo];
  for (int s = 0; s < ncol; ++s) a.out[s][i] = a.val[s][fr];
}

inline unsigned grid_for(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }
constexpr unsigned kWarpGrid = 8 * kNumSMs;     // warp-per-graph kernels: grid-stride over the graphs

}  // namespace csv
}  // namespace ddfa

extern "C" {

size_t ddfa_csv_index_workspace_bytes(int64_t nbytes) {
  if (nbytes < 0) return 0;
  const size_t c = (size_t)ddfa::csv::num_chunks(nbytes);
  return ddfa::csv::align16(sizeof(int32_t) * 3 * c) + sizeof(int64_t) * c;
}

int ddfa_csv_index_count(const uint8_t *text, int64_t nbytes, int64_t *info, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(nbytes >= 1 && text && info && workspace, "ddfa_csv_index_count: empty text or NULL pointer");
  DDFA_REQUIRE(aligned16(text) && aligned16(workspace), "ddfa_csv_index_count: text and workspace must be 16-byte aligned");
  DDFA_REQUIRE(num_chunks(nbytes) <= INT32_MAX, "ddfa_csv_index_count: %lld bytes is too long", (long long)nbytes);
  DDFA_REQUIRE(workspace_bytes >= ddfa_csv_index_workspace_bytes(nbytes), "ddfa_csv_index_count: workspace of %zu bytes, need %zu",
               workspace_bytes, ddfa_csv_index_workspace_bytes(nbytes));
  cudaStream_t stream = as_stream(stream_);
  const int64_t c = num_chunks(nbytes);
  int32_t *qpar = static_cast<int32_t *>(workspace), *cnt0 = qpar + c, *cnt1 = cnt0 + c;
  int64_t *off = reinterpret_cast<int64_t *>(static_cast<char *>(workspace) + align16(sizeof(int32_t) * 3 * c));
  index_count_kernel<<<(unsigned)c, kThreads, 0, stream>>>(text, nbytes, qpar, cnt0, cnt1);
  DDFA_CHECK_LAUNCH("index_count_kernel");
  index_scan_kernel<<<1, kThreads, 0, stream>>>(qpar, cnt0, cnt1, c, off, info);
  DDFA_CHECK_LAUNCH("index_scan_kernel");
  return DDFA_OK;
}

int ddfa_csv_index_rows(const uint8_t *text, int64_t nbytes, int64_t *row_end, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(nbytes >= 1 && text && row_end && workspace, "ddfa_csv_index_rows: empty text or NULL pointer");
  DDFA_REQUIRE(aligned16(text) && aligned16(workspace), "ddfa_csv_index_rows: text and workspace must be 16-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_csv_index_workspace_bytes(nbytes), "ddfa_csv_index_rows: workspace of %zu bytes, need %zu",
               workspace_bytes, ddfa_csv_index_workspace_bytes(nbytes));
  const int64_t c = num_chunks(nbytes);
  const int32_t *pin = static_cast<const int32_t *>(workspace);
  const int64_t *off = reinterpret_cast<const int64_t *>(static_cast<const char *>(workspace) + align16(sizeof(int32_t) * 3 * c));
  index_scatter_kernel<<<(unsigned)c, kThreads, 0, as_stream(stream_)>>>(text, nbytes, pin, off, row_end);
  DDFA_CHECK_LAUNCH("index_scatter_kernel");
  return DDFA_OK;
}

int ddfa_csv_fields(const uint8_t *text, const int64_t *row_end, int64_t rows, const int32_t *columns, int32_t num_columns,
                    int64_t *const *out, int64_t *info, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(rows >= 1 && text && row_end && columns && out && info, "ddfa_csv_fields: no rows or NULL pointer");
  DDFA_REQUIRE(num_columns >= 1 && num_columns <= DDFA_CSV_MAX_COLS, "ddfa_csv_fields: %d columns outside [1, %d]", num_columns,
               DDFA_CSV_MAX_COLS);
  DDFA_REQUIRE(rows - 1 < ((int64_t)1 << 55), "ddfa_csv_fields: %lld rows", (long long)rows);
  FieldArgs a = {};
  for (int s = 0; s < num_columns; ++s) {
    DDFA_REQUIRE(columns[s] >= 0 && (s == 0 || columns[s] > columns[s - 1]), "ddfa_csv_fields: columns must be ascending and >= 0");
    DDFA_REQUIRE(out[s] != nullptr || rows == 1, "ddfa_csv_fields: NULL output %d", s);
    a.col[s] = columns[s];
    a.out[s] = out[s];
  }
  cudaStream_t stream = as_stream(stream_);
  fields_init_kernel<<<1, 32, 0, stream>>>(info, num_columns);
  DDFA_CHECK_LAUNCH("fields_init_kernel");
  if (rows > 1) {
    fields_kernel<<<grid_for(rows - 1), kThreads, 0, stream>>>(text, row_end, rows - 1, a, num_columns, info);
    DDFA_CHECK_LAUNCH("fields_kernel");
  }
  return DDFA_OK;
}

size_t ddfa_row_sort_workspace_bytes(int32_t n) {
  if (n < 0) return 0;
  ddfa::csv::SortWs w;
  return ddfa::csv::sort_layout(n, nullptr, &w);
}

int ddfa_row_sort(const int64_t *major, int64_t major_min, int32_t major_bits, const int64_t *minor, int64_t minor_min, int32_t minor_bits,
                  int32_t n, int32_t *perm, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(n >= 1 && perm && workspace && major, "ddfa_row_sort: n=%d < 1 or NULL pointer", n);
  DDFA_REQUIRE(major_bits >= 0 && major_bits <= 64 && minor_bits >= 0 && minor_bits <= 64 && (minor || minor_bits == 0),
               "ddfa_row_sort: key bits outside [0, 64]");
  DDFA_REQUIRE(aligned16(workspace), "ddfa_row_sort: workspace must be 16-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_row_sort_workspace_bytes(n), "ddfa_row_sort: workspace of %zu bytes, need %zu", workspace_bytes,
               ddfa_row_sort_workspace_bytes(n));
  cudaStream_t stream = as_stream(stream_);
  SortWs w;
  sort_layout(n, workspace, &w);
  const int minor_passes = (minor_bits + 7) / 8, passes = minor_passes + (major_bits + 7) / 8;
  int32_t *buf[2] = {passes % 2 ? w.tmp : perm, passes % 2 ? perm : w.tmp};     // the last pass writes perm
  iota_kernel<<<grid_for(n), kThreads, 0, stream>>>(buf[0], n);
  DDFA_CHECK_LAUNCH("iota_kernel");
  const int32_t tiles = (int32_t)num_tiles(n);
  for (int p = 0; p < passes; ++p) {
    const bool mi = p < minor_passes;
    const int64_t *key = mi ? minor : major;
    const int64_t kmin = mi ? minor_min : major_min;
    const int shift = 8 * (mi ? p : p - minor_passes);
    sort_count_kernel<<<tiles, kThreads, 0, stream>>>(buf[p & 1], n, key, kmin, shift, tiles, w.counts);
    DDFA_CHECK_LAUNCH("sort_count_kernel");
    sort_scan_kernel<<<kBins, kThreads, 0, stream>>>(w.counts, tiles, w.row_total);
    DDFA_CHECK_LAUNCH("sort_scan_kernel");
    sort_scatter_kernel<<<tiles, kThreads, 0, stream>>>(buf[p & 1], n, key, kmin, shift, tiles, w.counts, w.row_total, buf[(p + 1) & 1]);
    DDFA_CHECK_LAUNCH("sort_scatter_kernel");
  }
  return DDFA_OK;
}

size_t ddfa_csv_graphs_workspace_bytes(int32_t node_rows) {
  if (node_rows < 0) return 0;
  ddfa::csv::GraphWs w;
  return ddfa::csv::graph_layout(node_rows, nullptr, &w);
}

int ddfa_csv_graphs(const int64_t *node_gid, const int32_t *node_perm, int32_t node_rows, const int64_t *edge_gid, const int32_t *edge_perm,
                    int32_t edge_rows, const int64_t *innode, const int64_t *outnode, int64_t *info, void *workspace, size_t workspace_bytes,
                    void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(node_rows >= 1 && edge_rows >= 0, "ddfa_csv_graphs: node_rows=%d, edge_rows=%d", node_rows, edge_rows);
  DDFA_REQUIRE(node_gid && node_perm && info && workspace && (edge_rows == 0 || (edge_gid && edge_perm && innode && outnode)),
               "ddfa_csv_graphs: NULL pointer");
  DDFA_REQUIRE(aligned16(workspace), "ddfa_csv_graphs: workspace must be 16-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_csv_graphs_workspace_bytes(node_rows), "ddfa_csv_graphs: workspace of %zu bytes, need %zu",
               workspace_bytes, ddfa_csv_graphs_workspace_bytes(node_rows));
  cudaStream_t stream = as_stream(stream_);
  GraphWs w;
  graph_layout(node_rows, workspace, &w);
  const bool multi = node_rows > 4 * 4096;
  DDFA_CUDA(cudaMemsetAsync(info, 0, sizeof(int64_t) * DDFA_CSV_GRAPH_INFO_WORDS, stream));
  DDFA_CUDA(cudaMemsetAsync(info + 2, 0xff, sizeof(int64_t), stream));
  DDFA_CUDA(cudaMemsetAsync(w.eoff, 0, sizeof(int32_t) * ((size_t)node_rows + 1), stream));
  head_kernel<<<grid_for(node_rows), kThreads, 0, stream>>>(node_gid, node_perm, node_rows, w.gidx);
  DDFA_CHECK_LAUNCH("head_kernel");
  int rc = scan_counts(w.gidx, nullptr, node_rows, multi ? w.sums0 : nullptr, nullptr, stream);
  if (rc != DDFA_OK) return rc;
  node_off_kernel<<<grid_for(node_rows), kThreads, 0, stream>>>(node_gid, node_perm, node_rows, w.gidx, w.node_off);
  DDFA_CHECK_LAUNCH("node_off_kernel");
  graph_kernel<<<kWarpGrid, kThreads, 0, stream>>>(node_gid, node_perm, node_rows, edge_gid, edge_perm, edge_rows, innode, outnode, w, info);
  DDFA_CHECK_LAUNCH("graph_kernel");
  graph_info_kernel<<<1, 1, 0, stream>>>(node_gid, node_perm, w, node_rows, info);
  DDFA_CHECK_LAUNCH("graph_info_kernel");
  rc = scan_counts(w.eoff, nullptr, node_rows, multi ? w.sums1 : nullptr, nullptr, stream);
  return rc;
}

int ddfa_csv_union(const int64_t *node_gid, const int32_t *node_perm, int32_t node_rows, const int64_t *vuln_col, const int32_t *edge_perm,
                   const int64_t *innode, const int64_t *outnode, int32_t num_graphs, const void *workspace, size_t workspace_bytes,
                   int32_t *src, int32_t *dst, int32_t *vuln, int64_t *nodes_per_graph, int64_t *edges_per_graph, int64_t *graph_ids,
                   void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(node_rows >= 1 && num_graphs >= 1 && num_graphs <= node_rows, "ddfa_csv_union: node_rows=%d, num_graphs=%d", node_rows,
               num_graphs);
  DDFA_REQUIRE(node_gid && node_perm && vuln_col && edge_perm && innode && outnode && workspace && src && dst && vuln && nodes_per_graph &&
                   edges_per_graph && graph_ids,
               "ddfa_csv_union: NULL pointer");
  DDFA_REQUIRE(workspace_bytes >= ddfa_csv_graphs_workspace_bytes(node_rows), "ddfa_csv_union: workspace of %zu bytes, need %zu",
               workspace_bytes, ddfa_csv_graphs_workspace_bytes(node_rows));
  cudaStream_t stream = as_stream(stream_);
  GraphWs w;
  graph_layout(node_rows, const_cast<void *>(workspace), &w);
  union_kernel<<<kWarpGrid, kThreads, 0, stream>>>(node_gid, node_perm, edge_perm, innode, outnode, w, num_graphs, src, dst, nodes_per_graph,
                                                   edges_per_graph, graph_ids);
  DDFA_CHECK_LAUNCH("union_kernel");
  vuln_kernel<<<grid_for(node_rows), kThreads, 0, stream>>>(vuln_col, node_perm, node_rows, vuln);
  DDFA_CHECK_LAUNCH("vuln_kernel");
  return DDFA_OK;
}

size_t ddfa_csv_join_workspace_bytes(int32_t feature_rows) {
  if (feature_rows < 0) return 0;
  return 2 * ddfa::csv::align16(sizeof(int64_t) * (size_t)feature_rows);
}

int ddfa_csv_join(const int64_t *node_gid, const int64_t *node_nid, const int32_t *node_perm, int32_t node_rows, const int64_t *feat_gid,
                  const int64_t *feat_nid, const int32_t *feat_perm, int32_t feature_rows, const int64_t *const *values, int32_t num_values,
                  int64_t *const *out, int64_t *info, void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::csv;
  DDFA_REQUIRE(node_rows >= 1 && feature_rows >= 0, "ddfa_csv_join: node_rows=%d, feature_rows=%d", node_rows, feature_rows);
  DDFA_REQUIRE(num_values >= 1 && num_values <= DDFA_CSV_MAX_COLS, "ddfa_csv_join: %d value columns outside [1, %d]", num_values,
               DDFA_CSV_MAX_COLS);
  DDFA_REQUIRE(node_gid && node_nid && node_perm && values && out && info && (feature_rows == 0 || (feat_gid && feat_nid && feat_perm && workspace)),
               "ddfa_csv_join: NULL pointer");
  DDFA_REQUIRE(workspace_bytes >= ddfa_csv_join_workspace_bytes(feature_rows), "ddfa_csv_join: workspace of %zu bytes, need %zu",
               workspace_bytes, ddfa_csv_join_workspace_bytes(feature_rows));
  JoinArgs a = {};
  for (int s = 0; s < num_values; ++s) {
    DDFA_REQUIRE(out[s] && (values[s] || feature_rows == 0), "ddfa_csv_join: NULL column %d", s);
    a.val[s] = values[s];
    a.out[s] = out[s];
  }
  cudaStream_t stream = as_stream(stream_);
  int64_t *sg = static_cast<int64_t *>(workspace);
  int64_t *sk = feature_rows ? reinterpret_cast<int64_t *>(static_cast<char *>(workspace) + align16(sizeof(int64_t) * (size_t)feature_rows))
                             : nullptr;
  DDFA_CUDA(cudaMemsetAsync(info, 0xff, sizeof(int64_t), stream));
  if (feature_rows) {
    join_keys_kernel<<<grid_for(feature_rows), kThreads, 0, stream>>>(feat_gid, feat_nid, feat_perm, feature_rows, sg, sk);
    DDFA_CHECK_LAUNCH("join_keys_kernel");
  }
  join_kernel<<<grid_for(node_rows), kThreads, 0, stream>>>(node_gid, node_nid, node_perm, node_rows, sg, sk, feat_perm, feature_rows, a,
                                                            num_values, info);
  DDFA_CHECK_LAUNCH("join_kernel");
  return DDFA_OK;
}

}  // extern "C"
