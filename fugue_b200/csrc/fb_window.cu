// K9  segmented inclusive scan: the window functions of a ColumnMap over the logical partitions of
// fa.transform (running / partition-wide aggregates, ranks).  The reference runs these as a pandas
// function per logical partition (fugue/execution/native_execution_engine.py:156-164).
//
// Reduce-then-scan in three launches, every combination in a fixed order so that results (f64 SUM
// included) are bit-identical from run to run:
//   1. one CTA per tile of kTile rows: the tile's segmented aggregate (a head inside the tile drops what
//      came before it) -> scratch
//   2. one CTA per column: exclusive segmented scan over the tile aggregates, in tile order -> the
//      carry into every tile (written over the aggregates)
//   3. one CTA per tile: the tile's scan again, started from its carry; writes value and count
// A decoupled look-back would read the inputs once instead of twice, but it combines inclusive
// prefixes or aggregates depending on timing, which changes the rounding of a float sum between runs.
// Segment heads never exist as a per-row array in HBM: a tile binary-searches the segment offsets
// for its first row and marks the heads that fall inside it in shared memory.
#include "fb_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;                  // consecutive rows per thread
constexpr int kTile = kThreads * kItems;   // rows per CTA
constexpr int kCarryThreads = 1024;

// one 8-byte pad word per kItems words: a thread reading its kItems consecutive rows from shared memory
// and a warp storing striped rows both hit distinct banks
__host__ __device__ constexpr int padded(int j) { return j + (j >> 3); }
static_assert(kItems == 8, "padded() assumes 8 rows per thread");

struct ScanCols {
  const void* vals[FB_SCAN_MAX_COLS];
  const uint8_t* valid[FB_SCAN_MAX_COLS];
  void* out_vals[FB_SCAN_MAX_COLS];
  int64_t* out_count[FB_SCAN_MAX_COLS];
  int32_t op[FB_SCAN_MAX_COLS];
  int32_t ncols;
};

// (value, count of valid rows, "a segment starts in here") of a run of consecutive rows
struct St {
  uint64_t v;
  int64_t c;
  int32_t f;
};

// IEEE totalOrder as a signed integer order: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN
__device__ __forceinline__ int64_t total_order(uint64_t b) {
  const int64_t s = (int64_t)b;
  return s >= 0 ? s : s ^ 0x7FFFFFFFFFFFFFFFLL;
}

__device__ __forceinline__ uint64_t combine_values(int op, uint64_t a, uint64_t b) {
  switch (op) {
    case FB_AGG_SUM_F64:
      return (uint64_t)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
    case FB_AGG_SUM_I64: return a + b;  // two's-complement wrap-around
    case FB_AGG_MIN_I64: return (int64_t)b < (int64_t)a ? b : a;
    case FB_AGG_MAX_I64: return (int64_t)b > (int64_t)a ? b : a;
    case FB_AGG_MIN_F64: return total_order(b) < total_order(a) ? b : a;
    case FB_AGG_MAX_F64: return total_order(b) > total_order(a) ? b : a;
    default: return 0;  // COUNT: only the count matters
  }
}

// `a` followed by `b`.  Runs without a valid row do not take part, so MIN / MAX need no identity value
// and the result is always one of the inputs' own bit patterns.
__device__ __forceinline__ St combine(int op, const St& a, const St& b) {
  if (b.f) return b;
  St r;
  r.f = a.f;
  r.c = a.c + b.c;
  r.v = a.c == 0 ? b.v : (b.c == 0 ? a.v : combine_values(op, a.v, b.v));
  return r;
}

__device__ __forceinline__ St shfl_up(const St& s, int d) {
  St r;
  r.v = __shfl_up_sync(0xFFFFFFFFu, (unsigned long long)s.v, d);
  r.c = __shfl_up_sync(0xFFFFFFFFu, (long long)s.c, d);
  r.f = __shfl_up_sync(0xFFFFFFFFu, s.f, d);
  return r;
}

// Exclusive scan of one state per thread across the CTA, and the CTA total; fixed combination order.
template <int kWarps>
__device__ __forceinline__ St block_exclusive(int op, const St& x, St* warp_tot, St* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  St inc = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const St o = shfl_up(inc, d);
    if (lane >= d) inc = combine(op, o, inc);
  }
  const St ex = shfl_up(inc, 1);
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  St pre{0, 0, 0}, tot{0, 0, 0};
  for (int i = 0; i < kWarps; ++i) {
    if (i == w) pre = tot;
    tot = combine(op, tot, warp_tot[i]);
  }
  *total = tot;
  __syncthreads();  // warp_tot is reused by the next call
  return lane == 0 ? pre : combine(op, pre, ex);
}

__device__ __forceinline__ int64_t upper_bound(const int64_t* __restrict__ a, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t m = (lo + hi) >> 1;
    if (__ldg(a + m) <= x) lo = m + 1; else hi = m;
  }
  return lo;
}

__device__ __forceinline__ int64_t lower_bound(const int64_t* __restrict__ a, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t m = (lo + hi) >> 1;
    if (__ldg(a + m) < x) lo = m + 1; else hi = m;
  }
  return lo;
}

struct TileSmem {
  uint64_t v[padded(kTile)];
  int64_t c[padded(kTile)];
  uint8_t valid[kTile];
  uint8_t head[kTile];
  St warp_tot[kThreads / 32];
  int64_t seg_range[2];
};

// kFinal = false: pass 1 (tile aggregates); true: pass 3 (outputs, from the carries of pass 2)
template <bool kFinal>
__global__ void __launch_bounds__(kThreads)
fb_segscan_tile_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                       const __grid_constant__ ScanCols a, int64_t ntiles, uint64_t* __restrict__ tile_v,
                       int64_t* __restrict__ tile_c, int32_t* __restrict__ tile_f) {
  __shared__ __align__(16) TileSmem sm;
  const int64_t tile = blockIdx.x;
  const int64_t start = tile * kTile;
  const int64_t end = start + kTile < nrows ? start + kTile : nrows;
  const int nloc = (int)(end - start);
  // ---- segment heads inside [start, end): offsets[s] for s in [segment of `start`, first offset >= end)
  for (int i = threadIdx.x; i < kTile; i += kThreads) sm.head[i] = 0;
  if (threadIdx.x == 0) {
    const int64_t s0 = upper_bound(offsets, nseg + 1, start) - 1;
    sm.seg_range[0] = s0 < 0 ? 0 : s0;
    sm.seg_range[1] = lower_bound(offsets, nseg + 1, end);
  }
  __syncthreads();
  for (int64_t s = sm.seg_range[0] + threadIdx.x; s < sm.seg_range[1]; s += kThreads) {
    const int64_t o = __ldg(offsets + s);
    if (o >= start && o < end) sm.head[o - start] = 1;
  }
  const int j0 = threadIdx.x * kItems;
  for (int col = 0; col < a.ncols; ++col) {
    const int op = a.op[col];
    const bool is_count = op == FB_AGG_COUNT;
    const uint64_t* __restrict__ src = (const uint64_t*)a.vals[col];
    const uint8_t* __restrict__ vm = a.valid[col];
    // striped (coalesced) loads into shared memory; rows past the end are invalid
    for (int i = threadIdx.x; i < kTile; i += kThreads) {
      const bool in = i < nloc;
      if (!is_count) sm.v[padded(i)] = in ? __ldg((const unsigned long long*)src + start + i) : 0;
      sm.valid[i] = in ? (vm == nullptr ? 1 : (__ldg(vm + start + i) != 0)) : 0;
    }
    __syncthreads();
    St acc{0, 0, 0};
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int j = j0 + k;
      const int c = sm.valid[j];
      const St x{c && !is_count ? sm.v[padded(j)] : 0, c, sm.head[j]};
      acc = combine(op, acc, x);
    }
    St total;
    const St pre = block_exclusive<kThreads / 32>(op, acc, sm.warp_tot, &total);
    if (!kFinal) {
      if (threadIdx.x == 0) {
        tile_v[col * ntiles + tile] = total.v;
        tile_c[col * ntiles + tile] = total.c;
        if (col == 0) tile_f[tile] = total.f;
      }
      continue;
    }
    St run = combine(op, St{tile_v[col * ntiles + tile], tile_c[col * ntiles + tile], 0}, pre);
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int j = j0 + k;
      const int c = sm.valid[j];
      const St x{c && !is_count ? sm.v[padded(j)] : 0, c, sm.head[j]};
      run = combine(op, run, x);
      sm.v[padded(j)] = run.c > 0 ? run.v : 0;  // no valid row yet: 0, not whatever preceded the segment
      sm.c[padded(j)] = run.c;
    }
    __syncthreads();
    uint64_t* __restrict__ ov = (uint64_t*)a.out_vals[col];
    int64_t* __restrict__ oc = a.out_count[col];
    for (int i = threadIdx.x; i < nloc; i += kThreads) {
      if (ov != nullptr) ov[start + i] = sm.v[padded(i)];
      if (oc != nullptr) oc[start + i] = sm.c[padded(i)];
    }
    __syncthreads();  // shared buffers are refilled by the next column
  }
}

// pass 2: per column, the exclusive segmented scan of the tile aggregates (in place: aggregate -> carry)
__global__ void __launch_bounds__(kCarryThreads)
fb_segscan_carry_kernel(int64_t ntiles, const __grid_constant__ ScanCols a, uint64_t* __restrict__ tile_v,
                        int64_t* __restrict__ tile_c, const int32_t* __restrict__ tile_f) {
  __shared__ St warp_tot[kCarryThreads / 32];
  const int col = blockIdx.x;
  const int op = a.op[col];
  uint64_t* tv = tile_v + col * ntiles;
  int64_t* tc = tile_c + col * ntiles;
  const int64_t per = (ntiles + kCarryThreads - 1) / kCarryThreads;
  const int64_t b = threadIdx.x * per;
  const int64_t e = b + per < ntiles ? b + per : ntiles;
  St acc{0, 0, 0};
  for (int64_t t = b; t < e; ++t) acc = combine(op, acc, St{tv[t], tc[t], tile_f[t]});
  St total;
  St run = block_exclusive<kCarryThreads / 32>(op, acc, warp_tot, &total);
  for (int64_t t = b; t < e; ++t) {
    const St x{tv[t], tc[t], tile_f[t]};
    tv[t] = run.v;
    tc[t] = run.c;
    run = combine(op, run, x);
  }
}

int64_t num_tiles(int64_t nrows) { return (nrows + kTile - 1) / kTile; }

}  // namespace

extern "C" size_t fb_segmented_scan_scratch_bytes(int64_t nrows, int ncols) {
  if (nrows <= 0 || ncols <= 0) return 0;
  return (size_t)num_tiles(nrows) * (16 * (size_t)ncols + 4);
}

extern "C" int fb_segmented_scan(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                 int ncols, const int32_t* ops, const void* const* vals,
                                 const uint8_t* const* valid, void* const* out_vals, int64_t* const* out_count,
                                 void* scratch, size_t scratch_bytes) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK(ncols >= 1 && ncols <= FB_SCAN_MAX_COLS, "ncols=%d out of range [1,%d]", ncols, FB_SCAN_MAX_COLS);
  FB_CHECK(ops != nullptr, "NULL ops");
  ScanCols a;
  memset(&a, 0, sizeof(a));
  a.ncols = ncols;
  for (int c = 0; c < ncols; ++c) {
    FB_CHECK(ops[c] >= FB_AGG_SUM_F64 && ops[c] <= FB_AGG_MAX_F64, "column %d: unknown scan op %d", c, ops[c]);
    a.op[c] = ops[c];
    a.vals[c] = vals != nullptr ? vals[c] : nullptr;
    a.valid[c] = valid != nullptr ? valid[c] : nullptr;
    a.out_vals[c] = out_vals != nullptr ? out_vals[c] : nullptr;
    a.out_count[c] = out_count != nullptr ? out_count[c] : nullptr;
    FB_CHECK(nrows == 0 || ops[c] == FB_AGG_COUNT || a.vals[c] != nullptr, "column %d: op %d needs a value column", c, ops[c]);
  }
  if (nrows == 0) return 0;
  FB_CHECK(nseg >= 1 && d_offsets != nullptr, "%lld rows need at least one segment", (long long)nrows);
  const int64_t ntiles = num_tiles(nrows);
  FB_CHECK(ntiles < (1LL << 31), "too many rows");
  FB_CHECK(scratch != nullptr && scratch_bytes >= fb_segmented_scan_scratch_bytes(nrows, ncols),
           "scratch too small: %zu < %zu", scratch_bytes, fb_segmented_scan_scratch_bytes(nrows, ncols));
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  uint64_t* tile_v = (uint64_t*)scratch;
  int64_t* tile_c = (int64_t*)(tile_v + ncols * ntiles);
  int32_t* tile_f = (int32_t*)(tile_c + ncols * ntiles);
  cudaStream_t st = (cudaStream_t)stream;
  fb_segscan_tile_kernel<false><<<(unsigned)ntiles, kThreads, 0, st>>>(nrows, nseg, d_offsets, a, ntiles, tile_v,
                                                                         tile_c, tile_f);
  FB_CUDA(cudaGetLastError());
  fb_segscan_carry_kernel<<<ncols, kCarryThreads, 0, st>>>(ntiles, a, tile_v, tile_c, tile_f);
  FB_CUDA(cudaGetLastError());
  fb_segscan_tile_kernel<true><<<(unsigned)ntiles, kThreads, 0, st>>>(nrows, nseg, d_offsets, a, ntiles, tile_v,
                                                                        tile_c, tile_f);
  FB_CUDA(cudaGetLastError());
  return 0;
}
