// K10  exact order statistics per segment: PERCENTILE_CONT / PERCENTILE_DISC / MEDIAN of a column over the
// logical partitions of fa.transform (window form) and over the groups of a sorted GROUP BY.
//
// Every segment's non-NULL values are ordered ascending (ties by row, NULL and NaN last, -0.0 equal to 0.0:
// the order of sort.argsort_rows), then each requested quantile is read at its sorted position.  Two paths,
// chosen per segment by its length alone:
//   - short (length <= FB_QUANTILE_TILE_ROWS = T): CTA t owns the segments that START in rows [tT, (t+1)T).
//     They span fewer than 2T rows.  The CTA stages (segment start, NULL flag, order key, row) as one
//     128-bit key per row in shared memory, bitonic-sorts them (the segment start is the most significant
//     field, so every segment stays in its own rows), and writes the per-segment results.  The column is
//     read once; nothing but the results goes back to HBM.
//   - long (length > T): a segment longer than T that starts in CTA t's window is the last one starting
//     there, so each CTA names at most one.  Their rows are gathered as (order key, row, long ordinal, NULL
//     flag) columns and sorted by the radix passes of the sort (fb_radix_pass: order key bytes, then the NULL
//     flag, then the ordinal; all stable, starting from row order), and a pick kernel reads the positions.
// Both paths order by the same key and pick with the same arithmetic, so they give identical results.
#include <mutex>

#include "fb_common.cuh"

namespace {

constexpr int kQThreads = 512;
constexpr int kTileRows = FB_QUANTILE_TILE_ROWS;
constexpr int kStage = 2 * kTileRows;  // staged rows of one CTA: < 2T
constexpr int kPickThreads = 256;
constexpr uint64_t kSign = 0x8000000000000000ULL;

static_assert(kStage <= (1 << 13), "row and segment offsets inside a CTA take 13 bits");

struct QSpec {
  double q[FB_QUANTILE_MAX_Q];
  int32_t kind[FB_QUANTILE_MAX_Q];
  void* out[FB_QUANTILE_MAX_Q];
  int32_t nq;
};

// the unsigned order key of sort._unsigned_order_key; false: the row is NULL (or a float NaN)
__device__ __forceinline__ bool order_key(const void* vals, const uint8_t* valid, int cls, int64_t row,
                                          uint64_t* key) {
  if (valid != nullptr && __ldg(valid + row) == 0) return false;
  uint64_t b = __ldg((const unsigned long long*)vals + row);
  if (cls == FB_RANGE_KEY_I64) {
    *key = b ^ kSign;
  } else if (cls == FB_RANGE_KEY_U64) {
    *key = b;
  } else {
    const double x = __longlong_as_double((long long)b);
    if (x != x) return false;
    if (x == 0.0) b = 0;
    *key = (int64_t)b < 0 ? ~b : b ^ kSign;
  }
  return true;
}

// a value as f64 by its class: uint64 converts as unsigned, the order the sort gives it
__device__ __forceinline__ double as_f64(const void* vals, int cls, int64_t row) {
  const uint64_t b = __ldg((const unsigned long long*)vals + row);
  if (cls == FB_RANGE_KEY_I64) return __ll2double_rn((long long)b);
  if (cls == FB_RANGE_KEY_U64) return __ull2double_rn((unsigned long long)b);
  return __longlong_as_double((long long)b);
}

// The results of one segment of m non-NULL values; row_at(p) is the row at sorted position p < m.
template <class RowAt>
__device__ __forceinline__ void pick(const QSpec& qs, const void* vals, int cls, int64_t seg, int64_t m,
                                     int64_t* count, RowAt row_at) {
  count[seg] = m;
  for (int j = 0; j < qs.nq; ++j) {
    const double q = qs.q[j];
    if (qs.kind[j] == FB_QUANTILE_DISC) {
      int64_t r = -1;
      if (m > 0) {
        int64_t p = (int64_t)ceil(__dmul_rn(q, (double)m)) - 1;
        p = p < 0 ? 0 : (p > m - 1 ? m - 1 : p);
        r = row_at(p);
      }
      ((int64_t*)qs.out[j])[seg] = r;
    } else {
      double v = 0.0;
      if (m > 0) {
        const double h = __dmul_rn(q, (double)(m - 1));
        const double lo = floor(h);
        const double frac = __dsub_rn(h, lo);
        int64_t p = (int64_t)lo;
        p = p > m - 1 ? m - 1 : p;
        v = as_f64(vals, cls, row_at(p));
        if (frac != 0.0 && p + 1 < m) {
          const double x1 = as_f64(vals, cls, row_at(p + 1));
          v = __dadd_rn(v, __dmul_rn(__dsub_rn(x1, v), frac));
        }
      }
      ((double*)qs.out[j])[seg] = v;
    }
  }
}

// first index of [0, n) with a[index] > x (a ascending)
__device__ __forceinline__ int64_t upper_bound(const int64_t* __restrict__ a, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (__ldg(a + m) <= x) lo = m + 1; else hi = m;
  }
  return lo;
}

// first index of [0, n) with a[index] >= x (a ascending)
__device__ __forceinline__ int64_t lower_bound(const int64_t* __restrict__ a, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (__ldg(a + m) < x) lo = m + 1; else hi = m;
  }
  return lo;
}

// The 128-bit sort key of a staged row: hi = segment start (13 bits) | NULL flag | order key >> 14,
// lo = order key << 50 | row (13 bits).  Padding is all ones and sorts after every row.
struct Key {
  unsigned long long hi, lo;
};

__device__ __forceinline__ bool key_gt(const Key& a, const Key& b) {
  return a.hi > b.hi || (a.hi == b.hi && a.lo > b.lo);
}

// Short path: one CTA per window of T rows (see the top of the file).  Also names the window's long segment
// (long_seg[t] = its id or -1, long_len[t] = its length or 0) for the long path.
__global__ void __launch_bounds__(kQThreads)
fb_quantile_short_kernel(int64_t nrows, int64_t nseg, int64_t ntiles, const int64_t* __restrict__ offsets,
                         const void* __restrict__ vals, const uint8_t* __restrict__ valid, int cls,
                         const __grid_constant__ QSpec qs, int64_t* __restrict__ count,
                         int64_t* __restrict__ long_flag, int64_t* __restrict__ long_len,
                         int64_t* __restrict__ long_seg) {
  extern __shared__ Key keys[];
  __shared__ int64_t win[4];  // first segment, end of the short segments, first row, staged rows
  const int64_t t = blockIdx.x;
  if (threadIdx.x == 0) {
    const int64_t s0 = lower_bound(offsets, nseg, t * kTileRows);
    int64_t s1 = t == ntiles - 1 ? nseg : lower_bound(offsets, nseg, (t + 1) * kTileRows);
    int64_t lseg = -1, llen = 0;
    if (s1 > s0) {
      const int64_t len = __ldg(offsets + s1) - __ldg(offsets + s1 - 1);
      if (len > kTileRows) {
        lseg = s1 - 1;
        llen = len;
        --s1;
      }
    }
    long_flag[t] = lseg >= 0 ? 1 : 0;
    long_len[t] = llen;
    long_seg[t] = lseg;
    win[0] = s0;
    win[1] = s1;
    win[2] = __ldg(offsets + s0);
    win[3] = __ldg(offsets + s1) - win[2];
  }
  __syncthreads();
  const int64_t s0 = win[0], s1 = win[1], r0 = win[2];
  const int L = (int)win[3];
  if (s1 <= s0) return;
  int P = 1;
  while (P < L) P <<= 1;
  for (int j = threadIdx.x; j < P; j += kQThreads) {
    Key k{~0ULL, ~0ULL};
    if (j < L) {
      const int64_t row = r0 + j;
      const int64_t s = s0 + upper_bound(offsets + s0, s1 - s0, row) - 1;
      const uint64_t start = (uint64_t)(__ldg(offsets + s) - r0);
      uint64_t ok = 0;
      const uint64_t null = order_key(vals, valid, cls, row, &ok) ? 0 : 1;
      k.hi = (start << 51) | (null << 50) | (ok >> 14);
      k.lo = (ok << 50) | (uint64_t)j;
    }
    keys[j] = k;
  }
  __syncthreads();
  // bitonic sort of P keys, P / 2 compare-exchanges per step
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (P >> 1); i += kQThreads) {
        const int a = 2 * i - (i & (stride - 1));
        const int b = a + stride;
        const Key x = keys[a], y = keys[b];
        if (key_gt(x, y) == ((a & size) == 0)) {
          keys[a] = y;
          keys[b] = x;
        }
      }
      __syncthreads();
    }
  }
  for (int64_t s = s0 + threadIdx.x; s < s1; s += kQThreads) {
    const int a = (int)(__ldg(offsets + s) - r0), b = (int)(__ldg(offsets + s + 1) - r0);
    int lo = a, hi = b;  // the first NULL of the segment's sorted rows
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if ((keys[m].hi >> 50) & 1) hi = m; else lo = m + 1;
    }
    pick(qs, vals, cls, s, (int64_t)(lo - a), count,
         [&](int64_t p) { return r0 + (int64_t)(keys[a + p].lo & 0x1FFF); });
  }
}

// long path, 1: list the long segments in segment order: ordinal k -> segment id, first row in the gathered
// arrays (dst[nlong] = the number of gathered rows)
__global__ void fb_quantile_list_kernel(int64_t ntiles, const int64_t* __restrict__ flag,
                                        const int64_t* __restrict__ ord, const int64_t* __restrict__ dst,
                                        const int64_t* __restrict__ long_seg, const int64_t* __restrict__ totals,
                                        int64_t* __restrict__ lseg, int64_t* __restrict__ ldst) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < ntiles && flag[t]) {
    lseg[ord[t]] = long_seg[t];
    ldst[ord[t]] = dst[t];
  }
  if (t == 0) ldst[totals[0]] = totals[1];
}

// long path, 2: the long segments' rows as (order key, row, ordinal, NULL flag); NULL rows get key 0, so they
// keep row order.  mm[0] / mm[1]: min / max order key of the non-NULL rows, mm[2]: NULL rows.
__global__ void __launch_bounds__(kPickThreads)
fb_quantile_gather_kernel(int64_t nlong, int64_t rows, const int64_t* __restrict__ offsets,
                          const int64_t* __restrict__ lseg, const int64_t* __restrict__ ldst,
                          const void* __restrict__ vals, const uint8_t* __restrict__ valid, int cls,
                          uint64_t* __restrict__ okey, int64_t* __restrict__ idx, int64_t* __restrict__ ordinal,
                          int64_t* __restrict__ nullf, unsigned long long* __restrict__ mm) {
  const int64_t j = (int64_t)blockIdx.x * kPickThreads + threadIdx.x;
  if (j >= rows) return;
  const int64_t k = upper_bound(ldst, nlong + 1, j) - 1;
  const int64_t row = __ldg(offsets + __ldg(lseg + k)) + (j - __ldg(ldst + k));
  uint64_t ok = 0;
  const bool v = order_key(vals, valid, cls, row, &ok);
  okey[j] = ok;
  idx[j] = row;
  ordinal[j] = k;
  nullf[j] = v ? 0 : 1;
  if (v) {
    atomicMin(mm, (unsigned long long)ok);
    atomicMax(mm + 1, (unsigned long long)ok);
  } else {
    atomicAdd(mm + 2, 1ULL);
  }
}

// long path, 3: one thread per long segment reads its sorted positions
__global__ void __launch_bounds__(kPickThreads)
fb_quantile_pick_kernel(int64_t nlong, const int64_t* __restrict__ lseg, const int64_t* __restrict__ ldst,
                        const int64_t* __restrict__ idx, const int64_t* __restrict__ nullf,
                        const void* __restrict__ vals, int cls, const __grid_constant__ QSpec qs,
                        int64_t* __restrict__ count) {
  const int64_t k = (int64_t)blockIdx.x * kPickThreads + threadIdx.x;
  if (k >= nlong) return;
  const int64_t a = __ldg(ldst + k), b = __ldg(ldst + k + 1);
  int64_t lo = a, hi = b;
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (__ldg(nullf + m)) hi = m; else lo = m + 1;
  }
  pick(qs, vals, cls, __ldg(lseg + k), lo - a, count, [&](int64_t p) { return __ldg(idx + a + p); });
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int64_t num_tiles(int64_t nrows) { return nrows <= 0 ? 1 : (nrows + kTileRows - 1) / kTileRows; }

// scratch layout: per-window arrays, scan scratch, totals; then the long rows
struct Layout {
  size_t flag, len, seg, ord, dst, lseg, ldst, scan, totals, rows, total;
};

Layout layout(int dev, int64_t nrows, int64_t long_rows) {
  Layout L;
  const int64_t nt = num_tiles(nrows);
  const size_t w = align256((size_t)(nt + 1) * 8);
  size_t o = 0;
  L.flag = o; o += w;
  L.len = o; o += w;
  L.seg = o; o += w;
  L.ord = o; o += w;
  L.dst = o; o += w;
  L.lseg = o; o += w;
  L.ldst = o; o += w;
  L.scan = o; o += align256(fb_exclusive_scan_scratch_bytes(nt));
  L.totals = o; o += 256;
  L.rows = o;
  if (long_rows > 0) {
    // okey, idx, ordinal, NULL flag, twice (the passes ping-pong), radix digit offsets, radix scratch
    o += 8 * align256((size_t)long_rows * 8) + align256(257 * 8) +
         align256(fb_partition_scratch_bytes(dev, long_rows, 256));
  }
  L.total = o;
  return L;
}

int radix_pass(int dev, cudaStream_t st, int64_t n, const void* key, int shift, int ncols, void* const* in,
               void* const* out, void* scratch, size_t scratch_bytes, int64_t* offsets) {
  const int32_t widths[4] = {8, 8, 8, 8};
  return fb_radix_pass(dev, st, n, key, shift, ncols, (const void* const*)in, widths, out, scratch, scratch_bytes,
                       offsets);
}

int nbytes_of(uint64_t diff) {
  int b = 0;
  while (diff != 0) {
    ++b;
    diff >>= 8;
  }
  return b;
}

}  // namespace

extern "C" size_t fb_quantile_scratch_bytes(int dev, int64_t nrows, int64_t long_rows) {
  if (nrows < 0 || long_rows < 0) return 0;
  return layout(dev, nrows, long_rows).total;
}

extern "C" int fb_segmented_quantile(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                     const void* d_vals, const uint8_t* d_valid, int value_class, int nq,
                                     const double* qs, const int32_t* kinds, int64_t* d_count, void* const* outs,
                                     void* scratch, size_t scratch_bytes) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK(value_class == FB_RANGE_KEY_I64 || value_class == FB_RANGE_KEY_U64 || value_class == FB_RANGE_KEY_F64,
           "unknown value class %d", value_class);
  FB_CHECK(nq >= 1 && nq <= FB_QUANTILE_MAX_Q, "nq=%d out of range [1,%d]", nq, FB_QUANTILE_MAX_Q);
  FB_CHECK(qs != nullptr && kinds != nullptr && outs != nullptr, "NULL quantile arrays");
  QSpec spec;
  memset(&spec, 0, sizeof(spec));
  spec.nq = nq;
  for (int j = 0; j < nq; ++j) {
    FB_CHECK(qs[j] >= 0.0 && qs[j] <= 1.0, "quantile %d: q=%g outside [0, 1]", j, qs[j]);
    FB_CHECK(kinds[j] == FB_QUANTILE_CONT || kinds[j] == FB_QUANTILE_DISC, "quantile %d: unknown kind %d", j,
             kinds[j]);
    spec.q[j] = qs[j];
    spec.kind[j] = kinds[j];
    spec.out[j] = outs[j];
    FB_CHECK(nseg == 0 || outs[j] != nullptr, "quantile %d: NULL output", j);
  }
  if (nseg == 0) return 0;
  FB_CHECK(d_offsets != nullptr && d_count != nullptr, "NULL offsets or count");
  FB_CHECK(nrows == 0 || d_vals != nullptr, "NULL values");
  const int64_t nt = num_tiles(nrows);
  FB_CHECK(nt < (1LL << 31), "too many rows");
  const Layout base = layout(dev, nrows, 0);
  FB_CHECK(scratch != nullptr && scratch_bytes >= base.total, "scratch too small: %zu < %zu", scratch_bytes,
           base.total);
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  char* sc = (char*)scratch;
  int64_t* flag = (int64_t*)(sc + base.flag);
  int64_t* len = (int64_t*)(sc + base.len);
  int64_t* seg = (int64_t*)(sc + base.seg);
  {
    static std::mutex mu;
    static uint64_t optin_done = 0;
    std::lock_guard<std::mutex> lock(mu);
    if (!(dev >= 0 && dev < 64 && ((optin_done >> dev) & 1))) {
      FB_CUDA(cudaFuncSetAttribute(fb_quantile_short_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(kStage * sizeof(Key))));
      if (dev >= 0 && dev < 64) optin_done |= 1ull << dev;
    }
  }
  fb_quantile_short_kernel<<<(unsigned)nt, kQThreads, kStage * sizeof(Key), st>>>(
      nrows, nseg, nt, d_offsets, d_vals, d_valid, value_class, spec, d_count, flag, len, seg);
  FB_CUDA(cudaGetLastError());
  if (nrows <= kTileRows) return 0;  // no segment can be long
  // ---- long path: which segments, where their rows go
  int64_t* ord = (int64_t*)(sc + base.ord);
  int64_t* dst = (int64_t*)(sc + base.dst);
  int64_t* lseg = (int64_t*)(sc + base.lseg);
  int64_t* ldst = (int64_t*)(sc + base.ldst);
  int64_t* totals = (int64_t*)(sc + base.totals);  // nlong, long rows, min key, max key, NULL rows
  void* scan = sc + base.scan;
  const size_t scan_bytes = fb_exclusive_scan_scratch_bytes(nt);
  if (fb_exclusive_scan_i64(dev, st, nt, flag, ord, totals, scan, scan_bytes) != 0) return 2;
  if (fb_exclusive_scan_i64(dev, st, nt, len, dst, totals + 1, scan, scan_bytes) != 0) return 2;
  fb_quantile_list_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(nt, flag, ord, dst, seg, totals, lseg, ldst);
  FB_CUDA(cudaGetLastError());
  int64_t h[5];
  FB_CUDA(cudaMemcpyAsync(h, totals, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  FB_CUDA(cudaStreamSynchronize(st));
  const int64_t nlong = h[0], rows = h[1];
  if (nlong == 0) return 0;
  const Layout full = layout(dev, nrows, rows);
  FB_CHECK(scratch_bytes >= full.total, "scratch too small for %lld rows in segments longer than %d: %zu < %zu",
           (long long)rows, kTileRows, scratch_bytes, full.total);
  const size_t col = align256((size_t)rows * 8);
  char* r = sc + full.rows;
  void* bufs[2][4];
  for (int b = 0; b < 2; ++b)
    for (int c = 0; c < 4; ++c) bufs[b][c] = r + (size_t)(4 * b + c) * col;
  int64_t* digit_off = (int64_t*)(r + 8 * col);
  void* rscratch = r + 8 * col + align256(257 * 8);
  const size_t rscratch_bytes = align256(fb_partition_scratch_bytes(dev, rows, 256));
  const unsigned long long init[3] = {~0ULL, 0ULL, 0ULL};
  FB_CUDA(cudaMemcpyAsync(totals + 2, init, sizeof(init), cudaMemcpyHostToDevice, st));
  fb_quantile_gather_kernel<<<(unsigned)((rows + kPickThreads - 1) / kPickThreads), kPickThreads, 0, st>>>(
      nlong, rows, d_offsets, lseg, ldst, d_vals, d_valid, value_class, (uint64_t*)bufs[0][0], (int64_t*)bufs[0][1],
      (int64_t*)bufs[0][2], (int64_t*)bufs[0][3], (unsigned long long*)(totals + 2));
  FB_CUDA(cudaGetLastError());
  FB_CUDA(cudaMemcpyAsync(h + 2, totals + 2, 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  FB_CUDA(cudaStreamSynchronize(st));
  const uint64_t kmin = (uint64_t)h[2], kmax = (uint64_t)h[3];
  const int64_t nnull = h[4];
  // LSD passes, each stable: the order key's varying bytes, the NULL flag, the ordinal's bytes
  int cur = 0;
  const int key_bytes = kmin <= kmax ? nbytes_of(kmin ^ kmax) : 0;
  for (int b = 0; b < key_bytes; ++b, cur ^= 1) {
    if (radix_pass(dev, st, rows, bufs[cur][0], 8 * b, 4, bufs[cur], bufs[cur ^ 1], rscratch, rscratch_bytes,
                   digit_off) != 0)
      return 2;
  }
  // the order key is not needed any more: the remaining passes move (row, ordinal, NULL flag)
  if (nnull > 0) {
    if (radix_pass(dev, st, rows, bufs[cur][3], 0, 3, bufs[cur] + 1, bufs[cur ^ 1] + 1, rscratch, rscratch_bytes,
                   digit_off) != 0)
      return 2;
    cur ^= 1;
  }
  const int ord_bytes = nbytes_of((uint64_t)(nlong - 1));
  for (int b = 0; b < ord_bytes; ++b, cur ^= 1) {
    if (radix_pass(dev, st, rows, bufs[cur][2], 8 * b, 3, bufs[cur] + 1, bufs[cur ^ 1] + 1, rscratch,
                   rscratch_bytes, digit_off) != 0)
      return 2;
  }
  fb_quantile_pick_kernel<<<(unsigned)((nlong + kPickThreads - 1) / kPickThreads), kPickThreads, 0, st>>>(
      nlong, lseg, ldst, (const int64_t*)bufs[cur][1], (const int64_t*)bufs[cur][3], d_vals, value_class, spec,
      d_count);
  FB_CUDA(cudaGetLastError());
  return 0;
}
