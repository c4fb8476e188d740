// Threshold curves of a test pass on the device: the exact precision-recall and ROC curves, AUROC, average precision and the
// binned precision-recall curve of n stored probabilities and labels (layout and rules in include/ddfa_b200.h, K9''').
//
// Reference: BaseModule.test_epoch_end (base_module.py:348-383) runs torchmetrics < 0.10's PrecisionRecallCurve and
// BinnedPrecisionRecallCurve over test_preds / test_labels.  Their common core, _binary_clf_curve, sorts the probabilities in
// descending order and takes, at the last index of every run of equal values, the cumulative counts of positives (tps) and
// negatives (fps).  Here that is an LSD radix sort and a run-boundary scan:
//
//   key:     p -> the 32-bit key whose ascending order is p's descending order (-0.0 mapped to +0.0 first, since the reference
//            compares by difference and so ties them), the label carried alongside as one byte;
//   sort:    four passes of 8-bit digits, each a per-tile histogram, a scan of the histograms per digit across tiles, and a
//            stable scatter (warp-level __match_any_sync ranks, warps and tiles in order);
//   runs:    a sample ends a run when the next key differs; per-tile counts of run ends and positives, a one-CTA scan of them, and
//            an emit pass that writes (threshold, tps, fps) at each run end's compacted index.
//
// Every count is an integer, so the sort and the counts are the same in both DDFA_TUNE_DETERMINISTIC modes.  AUROC and average
// precision are fp64 sums: per-CTA partials over a grid that depends on n only (shuffle tree per warp, warps in order), added in
// CTA order by a one-thread launch, so they are bit-reproducible in both modes too.
#include <math.h>

#include "common.cuh"

namespace ddfa {
namespace curves {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kItems = 16;                    // samples per thread in a tile
constexpr int kTile = kThreads * kItems;      // 4096 samples per tile
constexpr int kWarpSpan = 32 * kItems;        // each warp owns 512 consecutive samples of its tile
constexpr int kBins = 256;                    // 8-bit digits
constexpr int kPasses = 4;
constexpr int kMaxCtas = 2 * kNumSMs;
enum { kDistinct = 0, kPrPoints = 1, kPositives = 2, kNegatives = 3, kNanProbs = 4, kBadLabels = 5, kOneClass = 6 };

inline int64_t num_tiles(int64_t n) { return (n + kTile - 1) / kTile; }
inline size_t align16(size_t b) { return (b + 15) & ~size_t(15); }

struct Workspace {
  double *partials;       // [2 * kMaxCtas]: AUROC and AP partials per CTA
  uint32_t *key[2];       // ping-pong key planes [n]
  uint8_t *lab[2];        // ping-pong label bytes [n] (1: positive)
  int64_t *counts;        // [kBins * tiles]: a digit's count per tile, then its exclusive prefix across tiles
  int64_t *row_total;     // [kBins]
  int64_t *tile_pos;      // [tiles]: positives per tile, then their exclusive prefix
  int64_t *tile_end;      // [tiles]: run ends per tile, then their exclusive prefix
};

// the workspace carved in order (base == nullptr: sizes only); returns the bytes it needs
inline size_t layout(int64_t n, void *base, Workspace *w) {
  const int64_t tiles = num_tiles(n);
  char *p = static_cast<char *>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) -> void * {
    void *q = p ? p + off : nullptr;
    off += align16(bytes);
    return q;
  };
  w->partials = static_cast<double *>(take(sizeof(double) * 2 * kMaxCtas));
  for (int i = 0; i < 2; ++i) w->key[i] = static_cast<uint32_t *>(take(sizeof(uint32_t) * (size_t)n));
  for (int i = 0; i < 2; ++i) w->lab[i] = static_cast<uint8_t *>(take((size_t)n));
  w->counts = static_cast<int64_t *>(take(sizeof(int64_t) * kBins * (size_t)tiles));
  w->row_total = static_cast<int64_t *>(take(sizeof(int64_t) * kBins));
  w->tile_pos = static_cast<int64_t *>(take(sizeof(int64_t) * (size_t)tiles));
  w->tile_end = static_cast<int64_t *>(take(sizeof(int64_t) * (size_t)tiles));
  return off;
}

// p -> key, ascending key order = descending p order; -0.0 is keyed as +0.0 (NaN keeps its bits)
__device__ __forceinline__ uint32_t desc_key(float p) {
  const uint32_t u = __float_as_uint(p == 0.f ? 0.f : p);
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}
// the inverse: the stored fp32 value, bit for bit (+0.0 for a zero)
__device__ __forceinline__ float key_value(uint32_t k) {
  const uint32_t asc = ~k;
  return __uint_as_float((asc & 0x80000000u) ? (asc & 0x7fffffffu) : ~asc);
}

// inclusive scan over the kThreads threads of a CTA (every thread calls it); total = the CTA's sum
__device__ __forceinline__ int64_t block_scan_incl(int64_t v, int64_t &total) {
  __shared__ int64_t s[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) s[warp] = v;
  __syncthreads();
  int64_t before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    const int64_t t = s[w];
    before += w < warp ? t : 0;
    total += t;
  }
  __syncthreads();
  return v + before;
}

// keys and label bytes; NaN probabilities and labels other than 0 / 1 counted into info
__global__ void __launch_bounds__(kThreads) key_kernel(const float *__restrict__ probs, const float *__restrict__ labels, int64_t n,
                                                       uint32_t *__restrict__ key, uint8_t *__restrict__ lab, int64_t *__restrict__ info) {
  int64_t nan_p = 0, bad = 0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const float p = probs[i], y = labels[i];
    key[i] = desc_key(p);
    lab[i] = y == 1.f ? 1 : 0;
    nan_p += isnan(p) ? 1 : 0;
    bad += (y == 0.f || y == 1.f) ? 0 : 1;
  }
  int64_t tn, tb;
  block_scan_incl(nan_p, tn);
  block_scan_incl(bad, tb);
  if (threadIdx.x == 0) {
    if (tn) atomicAdd(reinterpret_cast<unsigned long long *>(info + kNanProbs), (unsigned long long)tn);
    if (tb) atomicAdd(reinterpret_cast<unsigned long long *>(info + kBadLabels), (unsigned long long)tb);
  }
}

// the digit histogram of one tile -> counts[digit * tiles + tile]
__global__ void __launch_bounds__(kThreads) digit_count_kernel(const uint32_t *__restrict__ key, int64_t n, int shift, int64_t tiles,
                                                               int64_t *__restrict__ counts) {
  __shared__ int32_t h[kBins];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = blockIdx.x * (int64_t)kTile;
#pragma unroll 4
  for (int k = 0; k < kItems; ++k) {
    const int64_t i = base + k * kThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[(key[i] >> shift) & (kBins - 1)], 1);
  }
  __syncthreads();
  counts[threadIdx.x * tiles + blockIdx.x] = h[threadIdx.x];
}

// CTA per digit: its row of tile counts -> exclusive prefix across tiles (in place), its total -> row_total
__global__ void __launch_bounds__(kThreads) digit_scan_kernel(int64_t *__restrict__ counts, int64_t tiles, int64_t *__restrict__ row_total) {
  int64_t *row = counts + blockIdx.x * tiles;
  int64_t carry = 0;
  for (int64_t c0 = 0; c0 < tiles; c0 += kThreads) {
    const int64_t i = c0 + threadIdx.x;
    const int64_t v = i < tiles ? row[i] : 0;
    int64_t total;
    const int64_t incl = block_scan_incl(v, total);
    if (i < tiles) row[i] = carry + incl - v;
    carry += total;
  }
  if (threadIdx.x == 0) row_total[blockIdx.x] = carry;
}

// stable scatter of one tile by the digit at `shift`: a sample goes to digit base + the tile's prefix + the samples of its digit
// ahead of it in the tile (earlier warps, earlier rounds of its warp, lower lanes of its round)
__global__ void __launch_bounds__(kThreads) digit_scatter_kernel(const uint32_t *__restrict__ key_in, const uint8_t *__restrict__ lab_in,
                                                                 int64_t n, int shift, int64_t tiles, const int64_t *__restrict__ counts,
                                                                 const int64_t *__restrict__ row_total, uint32_t *__restrict__ key_out,
                                                                 uint8_t *__restrict__ lab_out) {
  __shared__ int64_t start[kWarps][kBins];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  const int64_t base = blockIdx.x * (int64_t)kTile + warp * kWarpSpan;
  for (int j = threadIdx.x; j < kWarps * kBins; j += kThreads) (&start[0][0])[j] = 0;
  __syncthreads();
  uint32_t k[kItems];
  uint8_t l[kItems];
  int d[kItems];
#pragma unroll
  for (int it = 0; it < kItems; ++it) {
    const int64_t i = base + it * 32 + lane;
    const bool valid = i < n;
    k[it] = valid ? key_in[i] : 0u;
    l[it] = valid ? lab_in[i] : 0;
    d[it] = valid ? (int)((k[it] >> shift) & (kBins - 1)) : kBins;
    const uint32_t peers = __match_any_sync(0xffffffffu, d[it]);
    if (valid && lane == __ffs(peers) - 1) start[warp][d[it]] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {
    // thread b: digit b's first position for this tile, then each warp's first position in warp order
    const int b = threadIdx.x;
    const int64_t tot = row_total[b];
    int64_t all;
    int64_t run = block_scan_incl(tot, all) - tot + counts[b * tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const int64_t c = start[w][b];
      start[w][b] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kItems; ++it) {
    const uint32_t peers = __match_any_sync(0xffffffffu, d[it]);
    if (d[it] < kBins) {
      const int64_t pos = start[warp][d[it]] + __popc(peers & lt);
      key_out[pos] = k[it];
      lab_out[pos] = l[it];
    }
    __syncwarp();
    if (d[it] < kBins && lane == __ffs(peers) - 1) start[warp][d[it]] += __popc(peers);
    __syncwarp();
  }
}

// sample i of the sorted planes: does it end a run of equal keys, is it positive
__device__ __forceinline__ void run_flags(const uint32_t *__restrict__ key, const uint8_t *__restrict__ lab, int64_t n, int64_t i,
                                          bool &end, bool &pos) {
  end = pos = false;
  if (i < n) {
    end = i == n - 1 || key[i] != key[i + 1];
    pos = lab[i] != 0;
  }
}

// per tile: run ends and positives
__global__ void __launch_bounds__(kThreads) run_tile_kernel(const uint32_t *__restrict__ key, const uint8_t *__restrict__ lab, int64_t n,
                                                            int64_t *__restrict__ tile_pos, int64_t *__restrict__ tile_end) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = blockIdx.x * (int64_t)kTile + warp * kWarpSpan;
  int64_t e = 0, p = 0;
  for (int it = 0; it < kItems; ++it) {
    bool end, pos;
    run_flags(key, lab, n, base + it * 32 + lane, end, pos);
    e += end;
    p += pos;
  }
  int64_t te, tp;
  block_scan_incl(e, te);
  block_scan_incl(p, tp);
  if (threadIdx.x == 0) {
    tile_end[blockIdx.x] = te;
    tile_pos[blockIdx.x] = tp;
  }
}

// one CTA: exclusive prefixes of the tile counts (in place) and the totals: distinct thresholds, positives, negatives, one class
__global__ void __launch_bounds__(kThreads) run_scan_kernel(int64_t *__restrict__ tile_pos, int64_t *__restrict__ tile_end, int64_t tiles,
                                                            int64_t n, int64_t *__restrict__ info) {
  int64_t carry_p = 0, carry_e = 0;
  for (int64_t c0 = 0; c0 < tiles; c0 += kThreads) {
    const int64_t i = c0 + threadIdx.x;
    const int64_t vp = i < tiles ? tile_pos[i] : 0, ve = i < tiles ? tile_end[i] : 0;
    int64_t tp, te;
    const int64_t ip = block_scan_incl(vp, tp), ie = block_scan_incl(ve, te);
    if (i < tiles) {
      tile_pos[i] = carry_p + ip - vp;
      tile_end[i] = carry_e + ie - ve;
    }
    carry_p += tp;
    carry_e += te;
  }
  if (threadIdx.x == 0) {
    info[kDistinct] = carry_e;
    info[kPositives] = carry_p;
    info[kNegatives] = n - carry_p;
    info[kOneClass] = (carry_p == 0 || carry_p == n) ? 1 : 0;
  }
}

// each run end i -> (thresholds, tps, fps)[j], j = the run ends before it: the value, the positives in [0, i], i + 1 - that
__global__ void __launch_bounds__(kThreads) run_emit_kernel(const uint32_t *__restrict__ key, const uint8_t *__restrict__ lab, int64_t n,
                                                            const int64_t *__restrict__ tile_pos, const int64_t *__restrict__ tile_end,
                                                            float *__restrict__ thresholds, int64_t *__restrict__ tps,
                                                            int64_t *__restrict__ fps) {
  __shared__ int32_t wsum[2][kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  const int64_t base = blockIdx.x * (int64_t)kTile + warp * kWarpSpan;
  uint32_t endm = 0, posm = 0;
  int32_t we = 0, wp = 0;
#pragma unroll
  for (int it = 0; it < kItems; ++it) {
    bool end, pos;
    run_flags(key, lab, n, base + it * 32 + lane, end, pos);
    endm |= (uint32_t)end << it;
    posm |= (uint32_t)pos << it;
    we += __popc(__ballot_sync(0xffffffffu, end));
    wp += __popc(__ballot_sync(0xffffffffu, pos));
  }
  if (lane == 0) {
    wsum[0][warp] = we;
    wsum[1][warp] = wp;
  }
  __syncthreads();
  int64_t e_run = tile_end[blockIdx.x], p_run = tile_pos[blockIdx.x];
  for (int w = 0; w < warp; ++w) {
    e_run += wsum[0][w];
    p_run += wsum[1][w];
  }
#pragma unroll
  for (int it = 0; it < kItems; ++it) {
    const bool end = (endm >> it) & 1u, pos = (posm >> it) & 1u;
    const uint32_t be = __ballot_sync(0xffffffffu, end), bp = __ballot_sync(0xffffffffu, pos);
    if (end) {
      const int64_t i = base + it * 32 + lane;
      const int64_t j = e_run + __popc(be & lt);
      const int64_t cum = p_run + __popc(bp & lt) + 1 * pos;
      thresholds[j] = key_value(key[i]);
      tps[j] = cum;
      fps[j] = i + 1 - cum;
    }
    e_run += __popc(be);
    p_run += __popc(bp);
  }
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the PR curve (truncated at full recall, reversed, then (1, 0)), the ROC curve (leading (0, 0) at thresholds[0] + 1), and per
// CTA the trapezoids of the ROC curve and the terms (r[k+1] - r[k]) * p[k] of the PR curve
__global__ void __launch_bounds__(kThreads) curve_kernel(const float *__restrict__ thr, const int64_t *__restrict__ tps,
                                                         const int64_t *__restrict__ fps, int64_t *__restrict__ info,
                                                         double *__restrict__ pr_precision, double *__restrict__ pr_recall,
                                                         float *__restrict__ pr_thresholds, double *__restrict__ roc_fpr,
                                                         double *__restrict__ roc_tpr, float *__restrict__ roc_thresholds,
                                                         double *__restrict__ partials) {
  __shared__ int64_t s_len;
  __shared__ double s[kWarps][2];
  const int64_t m = info[kDistinct], P = info[kPositives], Nn = info[kNegatives];
  if (threadIdx.x == 0) {
    // the first index where tps reaches its last value (tps is non-decreasing)
    int64_t lo = 0, hi = m - 1;
    while (lo < hi) {
      const int64_t mid = lo + (hi - lo) / 2;
      if (tps[mid] >= P) hi = mid;
      else lo = mid + 1;
    }
    s_len = lo + 1;
    if (blockIdx.x == 0) info[kPrPoints] = lo + 1;
  }
  __syncthreads();
  const int64_t L = s_len;
  const double dP = (double)P, dN = (double)Nn;
  double auc = 0.0, ap = 0.0;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j <= m; j += (int64_t)gridDim.x * kThreads) {
    const double x0 = j ? (Nn > 0 ? (double)fps[j - 1] / dN : 0.0) : 0.0;
    const double y0 = j ? (P > 0 ? (double)tps[j - 1] / dP : 0.0) : 0.0;
    roc_fpr[j] = x0;
    roc_tpr[j] = y0;
    roc_thresholds[j] = j ? thr[j - 1] : thr[0] + 1.f;
    if (j < m) {
      const double x1 = Nn > 0 ? (double)fps[j] / dN : 0.0, y1 = P > 0 ? (double)tps[j] / dP : 0.0;
      auc += (x1 - x0) * (y0 + y1) / 2.0;
    }
    if (j < L) {
      const int64_t q = L - 1 - j;
      const double prec = (double)tps[q] / (double)(tps[q] + fps[q]), rec = (double)tps[q] / dP;
      pr_precision[j] = prec;
      pr_recall[j] = rec;
      pr_thresholds[j] = thr[q];
      const double rec_next = q > 0 ? (double)tps[q - 1] / dP : 0.0;
      ap += (rec_next - rec) * prec;
    } else if (j == L) {
      pr_precision[j] = 1.0;
      pr_recall[j] = 0.0;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auc = warp_sum_f64(auc);
  ap = warp_sum_f64(ap);
  if (lane == 0) {
    s[warp][0] = auc;
    s[warp][1] = ap;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += s[w][threadIdx.x];
    partials[blockIdx.x * 2 + threadIdx.x] = t;
  }
}

// the partials in CTA order: summary = {AUROC (NaN with one class), AP (NaN without positives)}
__global__ void curve_finish_kernel(const double *__restrict__ partials, int ctas, const int64_t *__restrict__ info,
                                    double *__restrict__ summary) {
  double auc = 0.0, ap = 0.0;
  for (int c = 0; c < ctas; ++c) {
    auc += partials[2 * c];
    ap += partials[2 * c + 1];
  }
  summary[0] = info[kOneClass] ? (double)NAN : auc;
  summary[1] = info[kPositives] > 0 ? -ap : (double)NAN;
}

// thread i: TP / FP at p >= t[i] from the distinct thresholds (binary search for the last one >= t[i]), then the binned rule
__global__ void __launch_bounds__(kThreads) binned_kernel(const float *__restrict__ thr, const int64_t *__restrict__ tps,
                                                          const int64_t *__restrict__ fps, const int64_t *__restrict__ info,
                                                          const float *__restrict__ t, int32_t T, double *__restrict__ bin_precision,
                                                          double *__restrict__ bin_recall) {
  const int32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i > T) return;
  if (i == T) {
    bin_precision[T] = 1.0;
    bin_recall[T] = 0.0;
    return;
  }
  const int64_t m = info[kDistinct], P = info[kPositives];
  const float ti = t[i];
  int64_t lo = 0, hi = m;          // lo: the number of distinct thresholds >= ti
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (thr[mid] >= ti) lo = mid + 1;
    else hi = mid;
  }
  const double tp = lo ? (double)tps[lo - 1] : 0.0, fp = lo ? (double)fps[lo - 1] : 0.0, fn = (double)P - tp;
  bin_precision[i] = (tp + 1e-6) / (tp + fp + 1e-6);
  bin_recall[i] = tp / (tp + fn + 1e-6);
}

inline int curve_ctas(int64_t n) {
  const int64_t c = (n + 1 + kThreads - 1) / kThreads;
  return (int)(c < 1 ? 1 : (c > kMaxCtas ? kMaxCtas : c));
}

inline bool aligned8(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

}  // namespace curves
}  // namespace ddfa

extern "C" {

size_t ddfa_curve_workspace_bytes(int64_t n) {
  if (n < 0) return 0;
  ddfa::curves::Workspace w;
  return ddfa::curves::layout(n, nullptr, &w);
}

int ddfa_curve_sort(const float *probs, const float *labels, int64_t n, float *thresholds, int64_t *tps, int64_t *fps, int64_t *info,
                    void *workspace, size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::curves;
  DDFA_REQUIRE(n >= 1 && num_tiles(n) <= INT32_MAX, "ddfa_curve_sort: n=%lld outside [1, 2^31 * %d]", (long long)n, kTile);
  DDFA_REQUIRE(probs && labels && thresholds && tps && fps && info && workspace, "ddfa_curve_sort: NULL pointer");
  DDFA_REQUIRE(aligned8(tps) && aligned8(fps) && aligned8(info) && aligned16(workspace),
               "ddfa_curve_sort: tps, fps and info must be 8-byte aligned, workspace 16-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_curve_workspace_bytes(n), "ddfa_curve_sort: workspace of %zu bytes, need %zu", workspace_bytes,
               ddfa_curve_workspace_bytes(n));
  cudaStream_t stream = as_stream(stream_);
  Workspace w;
  layout(n, workspace, &w);
  const int64_t tiles = num_tiles(n);
  DDFA_CUDA(cudaMemsetAsync(info, 0, sizeof(int64_t) * DDFA_CURVE_INFO_WORDS, stream));
  const int64_t kb = (n + kThreads - 1) / kThreads;
  key_kernel<<<(unsigned)(kb < 4 * kNumSMs ? kb : 4 * kNumSMs), kThreads, 0, stream>>>(probs, labels, n, w.key[0], w.lab[0], info);
  DDFA_CHECK_LAUNCH("key_kernel");
  for (int pass = 0; pass < kPasses; ++pass) {
    const int src = pass & 1, dst = src ^ 1;
    digit_count_kernel<<<(unsigned)tiles, kThreads, 0, stream>>>(w.key[src], n, 8 * pass, tiles, w.counts);
    DDFA_CHECK_LAUNCH("digit_count_kernel");
    digit_scan_kernel<<<kBins, kThreads, 0, stream>>>(w.counts, tiles, w.row_total);
    DDFA_CHECK_LAUNCH("digit_scan_kernel");
    digit_scatter_kernel<<<(unsigned)tiles, kThreads, 0, stream>>>(w.key[src], w.lab[src], n, 8 * pass, tiles, w.counts, w.row_total,
                                                                   w.key[dst], w.lab[dst]);
    DDFA_CHECK_LAUNCH("digit_scatter_kernel");
  }
  // an even number of passes: the sorted planes are key[0] / lab[0]
  run_tile_kernel<<<(unsigned)tiles, kThreads, 0, stream>>>(w.key[0], w.lab[0], n, w.tile_pos, w.tile_end);
  DDFA_CHECK_LAUNCH("run_tile_kernel");
  run_scan_kernel<<<1, kThreads, 0, stream>>>(w.tile_pos, w.tile_end, tiles, n, info);
  DDFA_CHECK_LAUNCH("run_scan_kernel");
  run_emit_kernel<<<(unsigned)tiles, kThreads, 0, stream>>>(w.key[0], w.lab[0], n, w.tile_pos, w.tile_end, thresholds, tps, fps);
  DDFA_CHECK_LAUNCH("run_emit_kernel");
  return DDFA_OK;
}

int ddfa_curve_metrics(const float *thresholds, const int64_t *tps, const int64_t *fps, int64_t n, const float *bin_thresholds,
                       int32_t num_bins, double *pr_precision, double *pr_recall, float *pr_thresholds, double *roc_fpr, double *roc_tpr,
                       float *roc_thresholds, double *bin_precision, double *bin_recall, double *summary, int64_t *info, void *workspace,
                       size_t workspace_bytes, void *stream_) {
  using namespace ddfa;
  using namespace ddfa::curves;
  DDFA_REQUIRE(n >= 1 && num_tiles(n) <= INT32_MAX, "ddfa_curve_metrics: n=%lld outside [1, 2^31 * %d]", (long long)n, kTile);
  DDFA_REQUIRE(num_bins >= 0 && num_bins < INT32_MAX, "ddfa_curve_metrics: num_bins=%d < 0", num_bins);
  DDFA_REQUIRE(thresholds && tps && fps && pr_precision && pr_recall && pr_thresholds && roc_fpr && roc_tpr && roc_thresholds &&
                   bin_precision && bin_recall && summary && info && workspace && (bin_thresholds || num_bins == 0),
               "ddfa_curve_metrics: NULL pointer");
  DDFA_REQUIRE(aligned8(tps) && aligned8(fps) && aligned8(info) && aligned8(pr_precision) && aligned8(pr_recall) && aligned8(roc_fpr) &&
                   aligned8(roc_tpr) && aligned8(bin_precision) && aligned8(bin_recall) && aligned8(summary) && aligned16(workspace),
               "ddfa_curve_metrics: the int64 / fp64 arrays must be 8-byte aligned, workspace 16-byte aligned");
  DDFA_REQUIRE(workspace_bytes >= ddfa_curve_workspace_bytes(n), "ddfa_curve_metrics: workspace of %zu bytes, need %zu", workspace_bytes,
               ddfa_curve_workspace_bytes(n));
  cudaStream_t stream = as_stream(stream_);
  Workspace w;
  layout(n, workspace, &w);
  const int ctas = curve_ctas(n);
  curve_kernel<<<ctas, kThreads, 0, stream>>>(thresholds, tps, fps, info, pr_precision, pr_recall, pr_thresholds, roc_fpr, roc_tpr,
                                              roc_thresholds, w.partials);
  DDFA_CHECK_LAUNCH("curve_kernel");
  curve_finish_kernel<<<1, 1, 0, stream>>>(w.partials, ctas, info, summary);
  DDFA_CHECK_LAUNCH("curve_finish_kernel");
  binned_kernel<<<(unsigned)((num_bins + 1 + kThreads - 1) / kThreads), kThreads, 0, stream>>>(thresholds, tps, fps, info, bin_thresholds,
                                                                                              num_bins, bin_precision, bin_recall);
  DDFA_CHECK_LAUNCH("binned_kernel");
  return DDFA_OK;
}

}  // extern "C"
