// K7: hash equi-join on sm_90a (build / probe-count / scan / probe-write / gather).
//
// Replaces NativeExecutionEngine.join -> triad PandasUtils.join -> pd.merge
//   fugue/execution/native_execution_engine.py:230-241, schema rule fugue/dataframe/utils.py:152-226.
// NULL keys never match (fugue_test/execution_suite.py:533-543).
//
// Design: open-addressing multimap in HBM, 16-byte slots {key, build_row + 1}; a build row claims
// the first free slot of its probe sequence with one atomicCAS on the row word (duplicates simply
// take further slots, no key comparison while building).  Probing is linear from the same hash;
// pass 1 counts the matches of every probe row, an exclusive scan turns counts into output
// offsets, pass 2 writes (probe_row, build_row) index pairs, and a gather kernel materialises the
// output columns (probe-side indices are monotonic -> coalesced reads; build side is a random
// 8-byte gather).  Output order: probe-row major, deterministic for a given table.
// Algorithmic bytes (SURVEY.md 8d, config 5): 16 + 16 read + 24 written per output row.
#include "fb_common.cuh"
#include "fb_tree.cuh"

namespace {

struct Slot {
  uint64_t key;
  unsigned long long rowp1;  // 0 = empty
};

inline int64_t l2_batch_bytes() {  // table bytes worked on at a time
  return (int64_t)64 << 20;
}

// clears slots [slot0, slot0 + nslots); status is reset when it is passed
__global__ void fb_join_clear_kernel(Slot* __restrict__ table_all, int64_t slot0, int64_t nslots,
                                     int64_t* __restrict__ status) {
  Slot* __restrict__ table = table_all + slot0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nslots;
       i += (int64_t)gridDim.x * blockDim.x) {
    table[i].key = 0;
    table[i].rowp1 = 0;
  }
  if (status != nullptr && blockIdx.x == 0 && threadIdx.x < 4) status[threadIdx.x] = 0;
}

__global__ void __launch_bounds__(256)
fb_join_build_kernel(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ valid, int64_t n,
                     Slot* __restrict__ table, int64_t capacity, int64_t* __restrict__ status, FbDiv dv,
                     int64_t region_shift, const int64_t* __restrict__ part_off, int p0, int p1) {
  // region_shift >= 0: the table is cut into regions of 1 << region_shift slots, one per hash
  // partition of the (hash-partitioned) inputs, so build and probe sweep it region by region
  // part_off != nullptr: only the rows of hash partitions [p0, p1) (one launch per batch of regions)
  const int64_t mask = region_shift >= 0 ? (((int64_t)1 << region_shift) - 1) : capacity - 1;
  const int64_t row_lo = part_off != nullptr ? part_off[p0] : 0;
  const int64_t row_hi = part_off != nullptr ? part_off[p1] : n;
  for (int64_t i = row_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < row_hi;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (valid != nullptr && valid[i] == 0) continue;  // NULL keys never match: not inserted
    const uint64_t key = keys[i];
    uint64_t h = fb_fmix64(key);
    int64_t base = 0;
    if (region_shift >= 0) {
      base = (int64_t)fb_fastmod(fb_hash_single_u64(key), dv) << region_shift;
      h >>= 7;
    }
    int64_t s = (int64_t)(h & (uint64_t)mask);
    bool done = false;
    for (int64_t probe = 0; probe <= mask; ++probe) {
      if (table[base + s].rowp1 == 0 &&
          atomicCAS(&table[base + s].rowp1, 0ULL, (unsigned long long)(i + 1)) == 0ULL) {
        table[base + s].key = key;
        done = true;
        break;
      }
      s = (s + 1) & mask;
    }
    if (!done) status[0] = 1;
  }
}

// kWrite == false: counts[i] = matches of probe row i
// kWrite == true : (out_probe, out_build)[offsets[i] + j] = (i, build row of the j-th match);
//                  with `outer`, a probe row without a match emits one pair (i, -1)
template <bool kWrite>
__global__ void __launch_bounds__(256)
fb_join_probe_kernel(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ valid, int64_t n,
                     const Slot* __restrict__ table, int64_t capacity, int outer,
                     int64_t* __restrict__ counts, const int64_t* __restrict__ offsets,
                     int64_t* __restrict__ out_probe, int64_t* __restrict__ out_build, FbDiv dv,
                     int64_t region_shift, int64_t* __restrict__ first) {
  // `first` (optional): the count pass records the build row of the first match (-1: none); the
  // write pass then emits rows with exactly one output pair straight from it, without walking the
  // table again (the common foreign-key -> unique-key join never touches the table twice)
  const int64_t mask = region_shift >= 0 ? (((int64_t)1 << region_shift) - 1) : capacity - 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = 0;
    int64_t o = kWrite ? offsets[i] : 0;
    int64_t f = -1;
    if (kWrite && first != nullptr) {
      const int64_t cnt = counts[i];
      if (cnt == 0) continue;
      if (cnt == 1) {
        out_probe[o] = i;
        out_build[o] = first[i];
        continue;
      }
    }
    if (valid == nullptr || valid[i] != 0) {
      const uint64_t key = keys[i];
      uint64_t h = fb_fmix64(key);
      int64_t base = 0;
      if (region_shift >= 0) {
        base = (int64_t)fb_fastmod(fb_hash_single_u64(key), dv) << region_shift;
        h >>= 7;
      }
      int64_t s = (int64_t)(h & (uint64_t)mask);
      for (int64_t probe = 0; probe <= mask; ++probe) {
        const unsigned long long r = table[base + s].rowp1;
        if (r == 0) break;
        if (table[base + s].key == key) {
          if (kWrite) {
            out_probe[o + c] = i;
            out_build[o + c] = (int64_t)r - 1;
          } else if (c == 0) {
            f = (int64_t)r - 1;
          }
          ++c;
        }
        s = (s + 1) & mask;
      }
    }
    if (outer && c == 0) {
      if (kWrite) {
        out_probe[o] = i;
        out_build[o] = -1;
      }
      c = 1;
    }
    if (!kWrite) {
      counts[i] = c;
      if (first != nullptr) first[i] = f;
    }
  }
}

// marks build rows that were matched by some probe row (for right/full outer joins)
__global__ void fb_join_mark_kernel(const int64_t* __restrict__ build_idx, int64_t n, uint8_t* __restrict__ matched) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    if (build_idx[i] >= 0) matched[build_idx[i]] = 1;
}

// ---- exclusive scan of int64 (3 kernels: tile sums, scan of sums, tile scan) ------------------
constexpr int kScanBlock = 512;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanBlock * kScanItems;

__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t* s_warp, int64_t& total) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int64_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
    if (lane >= (unsigned)o) x += y;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  int64_t base = 0, tot = 0;
  for (unsigned w = 0; w < blockDim.x / 32; ++w) {
    int64_t t = s_warp[w];
    if (w < warp) base += t;
    tot += t;
  }
  __syncthreads();
  total = tot;
  return base + x - v;
}

__global__ void __launch_bounds__(kScanBlock)
fb_scan_tile_sums_kernel(const int64_t* __restrict__ in, int64_t n, int64_t* __restrict__ sums) {
  __shared__ int64_t s_warp[kScanBlock / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  int64_t v = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    int64_t i = base + (int64_t)k * kScanBlock + threadIdx.x;
    if (i < n) v += in[i];
  }
  int64_t total;
  block_exclusive_scan(v, s_warp, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanBlock)
fb_scan_sums_kernel(int64_t* __restrict__ sums, int64_t ntiles, int64_t* __restrict__ total_out) {
  __shared__ int64_t s_warp[kScanBlock / 32];
  int64_t carry = 0;
  for (int64_t b0 = 0; b0 < ntiles; b0 += kScanBlock) {
    int64_t i = b0 + threadIdx.x;
    int64_t v = i < ntiles ? sums[i] : 0;
    int64_t total;
    int64_t ex = block_exclusive_scan(v, s_warp, total);
    if (i < ntiles) sums[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) *total_out = carry;
}

__global__ void __launch_bounds__(kScanBlock)
fb_scan_tiles_kernel(const int64_t* __restrict__ in, int64_t n, const int64_t* __restrict__ sums,
                     int64_t* __restrict__ out) {
  __shared__ int64_t s_warp[kScanBlock / 32];
  // thread t owns kScanItems consecutive elements
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  int64_t v[kScanItems];
  int64_t sum = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    v[k] = base + k < n ? in[base + k] : 0;
    sum += v[k];
  }
  int64_t total;
  int64_t run = sums[blockIdx.x] + block_exclusive_scan(sum, s_warp, total);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
}

// ---- row gather ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fb_gather_rows_kernel(const void* const* __restrict__ src_cols, void* const* __restrict__ dst_cols,
                      const int32_t* __restrict__ widths, const uint8_t* const* __restrict__ src_valid,
                      uint8_t* const* __restrict__ dst_valid, const int64_t* __restrict__ idx, int64_t n) {
  const int c = blockIdx.y;
  const int w = widths[c];
  const uint8_t* sv = src_valid ? src_valid[c] : nullptr;
  uint8_t* dv = dst_valid ? dst_valid[c] : nullptr;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n;
       o += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx[o];
    const bool has = r >= 0;
    switch (w) {
      case 8: ((uint64_t*)dst_cols[c])[o] = has ? ((const uint64_t*)src_cols[c])[r] : 0; break;
      case 4: ((uint32_t*)dst_cols[c])[o] = has ? ((const uint32_t*)src_cols[c])[r] : 0; break;
      case 2: ((uint16_t*)dst_cols[c])[o] = has ? ((const uint16_t*)src_cols[c])[r] : 0; break;
      default: ((uint8_t*)dst_cols[c])[o] = has ? ((const uint8_t*)src_cols[c])[r] : 0; break;
    }
    if (dv != nullptr) dv[o] = has ? (sv != nullptr ? sv[r] : (uint8_t)1) : (uint8_t)0;
  }
}

// ---- row scatter: the inverse of the gather ----------------------------------------------------------
// One thread per source row moves that row of every column, so the permutation is read once for all of
// them.  idx is a permutation (the host passes argsort results), so every destination row is written once.
__global__ void __launch_bounds__(256)
fb_scatter_rows_kernel(const void* const* __restrict__ src_cols, void* const* __restrict__ dst_cols,
                       const int32_t* __restrict__ widths, const uint8_t* const* __restrict__ src_valid,
                       uint8_t* const* __restrict__ dst_valid, const int64_t* __restrict__ idx, int64_t n,
                       int ncols) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx[i];
    for (int c = 0; c < ncols; ++c) {
      switch (widths[c]) {
        case 8: ((uint64_t*)dst_cols[c])[r] = ((const uint64_t*)src_cols[c])[i]; break;
        case 4: ((uint32_t*)dst_cols[c])[r] = ((const uint32_t*)src_cols[c])[i]; break;
        case 2: ((uint16_t*)dst_cols[c])[r] = ((const uint16_t*)src_cols[c])[i]; break;
        default: ((uint8_t*)dst_cols[c])[r] = ((const uint8_t*)src_cols[c])[i]; break;
      }
      uint8_t* dv = dst_valid[c];
      if (dv != nullptr) {
        const uint8_t* sv = src_valid[c];
        dv[r] = sv != nullptr ? sv[i] : (uint8_t)1;
      }
    }
  }
}

// ---- as-of search: per left row, the one right row of its run it matches --------------------------------
// The right side is sorted by (key, as-of value); run r = rows [run_off[r], run_off[r + 1]) of one key, its as-of
// values as unsigned order codes that ascend within the run (PRECONDITION: the host passes the codes of an
// argsort_rows result; it is not checked).  Codes of one integer class differ by exactly the values' distance
// (a signed code is the value + 2^63 mod 2^64), so an integer distance is one unsigned 64-bit subtraction of the
// larger code minus the smaller, in [0, 2^64) and never wrapping; a float distance is one f64 subtraction.
constexpr uint64_t kAsofSign = 0x8000000000000000ull;

__device__ __forceinline__ double asof_f64(uint64_t code) {  // inverse of the float order code (sort.py)
  return __longlong_as_double((long long)((code & kAsofSign) ? (code ^ kAsofSign) : ~code));
}

// first position in [lo, hi) whose code is > x (kUpper) or >= x, hi if none
template <bool kUpper>
__device__ __forceinline__ int64_t asof_bound(const uint64_t* __restrict__ codes, int64_t lo, int64_t hi,
                                              uint64_t x) {
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    const uint64_t c = __ldg((const unsigned long long*)codes + m);
    if (kUpper ? c <= x : c < x) lo = m + 1; else hi = m;
  }
  return lo;
}

// distance of codes a <= b: cls FB_RANGE_KEY_F64 compares the f64 in `f`, the integer classes the exact `u`
struct AsofDist {
  uint64_t u;
  double f;
};

__device__ __forceinline__ AsofDist asof_dist(uint64_t a, uint64_t b, bool is_float) {
  AsofDist d{0, 0.0};
  if (!is_float) d.u = b - a;
  else if (a != b) d.f = asof_f64(b) - asof_f64(a);  // equal codes are distance 0, also for +-inf
  return d;
}

__device__ __forceinline__ bool asof_le(const AsofDist& a, const AsofDist& b, bool is_float) {
  return is_float ? a.f <= b.f : a.u <= b.u;
}

__global__ void __launch_bounds__(256)
fb_asof_search_kernel(int64_t n, const int64_t* __restrict__ run, const int64_t* __restrict__ run_off,
                      const uint64_t* __restrict__ left_codes, const uint8_t* __restrict__ left_valid,
                      const uint64_t* __restrict__ codes, const int64_t* __restrict__ rows, int cls, int direction,
                      int strict, int has_tol, uint64_t tol, int64_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t res = -1;
  const int64_t r = __ldg((const long long*)run + i);
  if (r >= 0 && (left_valid == nullptr || __ldg(left_valid + i) != 0)) {
    const bool is_float = cls == FB_RANGE_KEY_F64;
    const AsofDist limit{tol, __longlong_as_double((long long)tol)};
    const int64_t s = __ldg((const long long*)run_off + r), e = __ldg((const long long*)run_off + r + 1);
    const uint64_t x = __ldg((const unsigned long long*)left_codes + i);
    int64_t b = -1, f = -1;  // backward / forward candidate positions in the sorted run
    AsofDist db{0, 0.0}, df{0, 0.0};
    if (direction != FB_ASOF_FORWARD) {  // the last code <= x (< x when strict): the last such row in input order
      const int64_t p = (strict ? asof_bound<false>(codes, s, e, x) : asof_bound<true>(codes, s, e, x)) - 1;
      if (p >= s) {
        db = asof_dist(__ldg((const unsigned long long*)codes + p), x, is_float);
        if (!has_tol || asof_le(db, limit, is_float)) b = p;
      }
    }
    if (direction != FB_ASOF_BACKWARD) {  // the first code >= x (> x when strict): the first such row
      const int64_t q = strict ? asof_bound<true>(codes, s, e, x) : asof_bound<false>(codes, s, e, x);
      if (q < e) {
        df = asof_dist(x, __ldg((const unsigned long long*)codes + q), is_float);
        if (!has_tol || asof_le(df, limit, is_float)) f = q;
      }
    }
    // nearest: the backward candidate unless the forward one is strictly closer
    const int64_t pick = b < 0 ? f : (f < 0 || asof_le(db, df, is_float) ? b : f);
    if (pick >= 0) res = __ldg((const long long*)rows + pick);
  }
  out[i] = res;
}

// ---- range join: per left row, every interval of its run that holds its value ----------------------------
// The right side is sorted by (key, start); run r = rows [run_off[r], run_off[r + 1]).  `ends` holds every sorted
// row's end code with the sign bit flipped (so a signed compare orders the unsigned codes), and `tv` the levels
// >= 1 of the aligned MAX tree over `ends` (fb_window_tree, layout TreeLevels): node (l, m) is the largest
// end of rows [m 2^l, (m + 1) 2^l).  A row with value x has its candidates in [s, p), p the end of the rows whose
// start passes the lower test; the hits among them are the rows whose flipped end is >= t (the upper test).
struct RangeTree {
  const int64_t* ends;  // level 0
  const int64_t* tv;    // levels >= 1
};

__device__ __forceinline__ int64_t range_node(const RangeTree& T, const TreeLevels& L, int level, int64_t m) {
  return level == 0 ? __ldg((const long long*)T.ends + m) : __ldg((const long long*)T.tv + L.off[level] + m);
}

// the last row of [s, q) whose end is >= t, -1 if none: the blocks of [s, q)'s canonical decomposition from
// right to left (the right-hand blocks by rising level, then the left-hand ones by falling level), then down
// the first block that holds a hit, to its rightmost row.  O(log (q - s)).
__device__ __forceinline__ int64_t range_prev_hit(const RangeTree& T, const TreeLevels& L, int64_t s, int64_t q,
                                                  int64_t t) {
  int64_t lo = s, hi = q;
  int level = 0;
  uint64_t left_levels = 0;  // levels with a left-hand block: block ceil(s / 2^l) there
  int64_t b = -1;
  for (; lo < hi; ++level, lo >>= 1, hi >>= 1) {
    if ((hi & 1) && range_node(T, L, level, hi - 1) >= t) {
      b = hi - 1;
      break;
    }
    hi &= ~(int64_t)1;
    if (lo & 1) {
      left_levels |= 1ull << level;
      ++lo;
    }
  }
  if (b < 0) {
    while (left_levels != 0) {
      level = 63 - __clzll((long long)left_levels);
      left_levels &= ~(1ull << level);
      const int64_t m = (s + ((int64_t)1 << level) - 1) >> level;
      if (range_node(T, L, level, m) >= t) {
        b = m;
        break;
      }
    }
    if (b < 0) return -1;
  }
  for (; level > 0; --level) b = range_node(T, L, level - 1, 2 * b + 1) >= t ? 2 * b + 1 : 2 * b;
  return b;
}

// kEmit == false: counts[i] = the row's matches (1 for an unmatched row when outer).  kEmit == true: the same walk
// writes its (left row, right row) pairs into [offsets[i], offsets[i] + counts[i]) from the back, so they come out
// in ascending sorted position, which is (start, right input order).
template <bool kEmit>
__global__ void __launch_bounds__(256)
fb_range_join_kernel(int64_t n, const int64_t* __restrict__ run, const int64_t* __restrict__ run_off,
                     const uint64_t* __restrict__ left_codes, const uint8_t* __restrict__ left_valid,
                     const uint64_t* __restrict__ starts, const RangeTree T, const __grid_constant__ TreeLevels L,
                     const int64_t* __restrict__ rows, int closed, int outer, int64_t* __restrict__ counts,
                     const int64_t* __restrict__ offsets, int64_t* __restrict__ out_left,
                     int64_t* __restrict__ out_right) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t c = 0, o = 0;
  if (kEmit) {
    o = __ldg((const long long*)offsets + i) + __ldg((const long long*)counts + i);  // one past the row's last slot
  }
  const int64_t r = __ldg((const long long*)run + i);
  if (r >= 0 && (left_valid == nullptr || __ldg(left_valid + i) != 0)) {
    const uint64_t x = __ldg((const unsigned long long*)left_codes + i);
    const int64_t s = __ldg((const long long*)run_off + r), e = __ldg((const long long*)run_off + r + 1);
    // lower test start <= x (closed left: the first start > x ends the candidates) or start < x
    const int64_t p = (closed & FB_RANGE_CLOSED_LEFT) ? asof_bound<true>(starts, s, e, x)
                                                        : asof_bound<false>(starts, s, e, x);
    // upper test end >= x (closed right) or end >= x + 1; nothing is > the largest code
    if ((closed & FB_RANGE_CLOSED_RIGHT) || x != ~0ull) {
      const int64_t t = (int64_t)(((closed & FB_RANGE_CLOSED_RIGHT) ? x : x + 1) ^ kAsofSign);
      for (int64_t q = range_prev_hit(T, L, s, p, t); q >= 0; q = range_prev_hit(T, L, s, q, t)) {
        ++c;
        if (kEmit) {
          --o;
          out_left[o] = i;
          out_right[o] = __ldg((const long long*)rows + q);
        }
      }
    }
  }
  if (c == 0 && outer) {
    c = 1;
    if (kEmit) {
      --o;
      out_left[o] = i;
      out_right[o] = -1;
    }
  }
  if (!kEmit) counts[i] = c;
}

// ---- stream compaction: indices of the non-zero bytes of a mask, in order ---------------------
__global__ void __launch_bounds__(kScanBlock)
fb_mask_tile_counts_kernel(const uint8_t* __restrict__ mask, int64_t n, int64_t* __restrict__ counts) {
  __shared__ int64_t s_warp[kScanBlock / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  int64_t v = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    int64_t i = base + (int64_t)k * kScanBlock + threadIdx.x;
    if (i < n && mask[i] != 0) ++v;
  }
  int64_t total;
  block_exclusive_scan(v, s_warp, total);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanBlock)
fb_mask_write_kernel(const uint8_t* __restrict__ mask, int64_t n, const int64_t* __restrict__ tile_base,
                     int64_t* __restrict__ out_idx) {
  __shared__ int64_t s_warp[kScanBlock / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  int64_t cnt = 0;
  uint8_t m[kScanItems];
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    m[k] = base + k < n ? mask[base + k] : 0;
    cnt += m[k] != 0;
  }
  int64_t total;
  int64_t o = tile_base[blockIdx.x] + block_exclusive_scan(cnt, s_warp, total);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (m[k] != 0) out_idx[o++] = base + k;
}

inline int64_t region_shift_of(int64_t capacity, uint32_t num_parts) {
  if (num_parts <= 1) return -1;
  int64_t sh = 0;
  while (((int64_t)num_parts << sh) < capacity) ++sh;
  return sh;
}

inline unsigned grid_for(int dev, int64_t n, int per_sm = 8) {
  int64_t b = (n + 255) / 256;
  int64_t m = (int64_t)fb_sm_count(dev) * per_sm;
  if (b > m) b = m;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// =====================================================================================================
// K7 fast path (inner / left outer, one 8-byte key): 4-byte slots + fused probe / output assembly.
//
//   table     : uint32 slots holding build_row + 1 (0 = empty): a quarter of the 16-byte multimap, so four
//               times as many regions of the radix join stay L2-resident and clearing costs a quarter; a
//               build row is ONE 32-bit CAS (no key store) - keys are compared through the build key
//               column, whose partition is L2-resident too (the inputs are hash-partitioned)
//   pass A    : every probe row walks its chain once: match count + first match (4 + 4 bytes per row) and
//               the per-tile totals; one block scans the tile totals -> output size
//   pass B    : per tile of 4096 probe rows the output slots [tile_base, tile_base + total) are mapped back
//               to (probe row, k-th match) through shared memory, then ONE thread per OUTPUT row copies the
//               probe-side columns (coalesced) and gathers the build-side columns (random, L2-resident):
//               no (probe, build) index pairs are materialised and there is no separate gather pass.
// Output order: probe-row major, matches in chain order - deterministic for a given table.
// =====================================================================================================
constexpr int kJ2Block = 512, kJ2Items = 8, kJ2Tile = kJ2Block * kJ2Items;
constexpr uint32_t kJ2None = 0xFFFFFFFFu;
constexpr int kJ2MaxCols = 48;

struct J2Cols {
  const void* src[kJ2MaxCols];
  void* dst[kJ2MaxCols];
  const uint8_t* vsrc[kJ2MaxCols];  // build side only: source validity (or NULL)
  uint8_t* vdst[kJ2MaxCols];        // build side only: output validity (or NULL)
  int32_t width[kJ2MaxCols];
  int32_t n;
};

__device__ __forceinline__ void j2_locate(uint64_t key, const FbDiv& dv, int64_t region_shift, int64_t capacity,
                                          int64_t& base, int64_t& s, int64_t& mask) {
  const uint64_t h = fb_hash_single_u64(key);  // the partitioner's hash: region = partition id
  if (region_shift >= 0) {
    base = (int64_t)fb_fastmod(h, dv) << region_shift;
    mask = ((int64_t)1 << region_shift) - 1;
  } else {
    base = 0;
    mask = capacity - 1;
  }
  s = (int64_t)((h >> 10) & (uint64_t)mask);
}

__global__ void fb_join2_clear_kernel(uint32_t* __restrict__ table, int64_t slot0, int64_t nslots) {
  uint4* t4 = (uint4*)(table + slot0);  // regions are multiples of 4 slots and 16-byte aligned
  const int64_t n4 = nslots >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
    t4[i] = make_uint4(0, 0, 0, 0);
}

__global__ void __launch_bounds__(256)
fb_join2_build_kernel(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ valid, int64_t n,
                      uint32_t* __restrict__ table, int64_t capacity, int64_t* __restrict__ status, FbDiv dv,
                      int64_t region_shift, const int64_t* __restrict__ part_off, int p0, int p1) {
  // status[0] = 1: a row found no free slot in its region (skewed build side; the host redoes it with one
  // region).  status[1] = 1: two build rows hold the same key.  Every occupied slot an inserter walks
  // past is compared with its key, and of two equal keys the one that claims its slot later always
  // walks past the earlier one (same home slot, no deletions), so the flag is exact; when it stays 0
  // the probe may stop at the first match.
  const int64_t row_lo = part_off != nullptr ? part_off[p0] : 0;
  const int64_t row_hi = part_off != nullptr ? part_off[p1] : n;
  bool dup = false;
  for (int64_t i = row_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < row_hi;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (valid != nullptr && valid[i] == 0) continue;  // NULL keys never match: not inserted
    const uint64_t key = keys[i];
    int64_t base, s, mask;
    j2_locate(key, dv, region_shift, capacity, base, s, mask);
    bool done = false;
    for (int64_t probe = 0; probe <= mask; ++probe) {
      uint32_t* slot = table + base + s;
      uint32_t e = *(volatile uint32_t*)slot;
      if (e == 0) {
        e = atomicCAS(slot, 0u, (uint32_t)(i + 1));
        if (e == 0u) {
          done = true;
          break;
        }
      }
      if (keys[e - 1] == key) dup = true;
      s = (s + 1) & mask;
    }
    if (!done) status[0] = 1;
  }
  if (dup) status[1] = 1;
}

// pass A
__global__ void __launch_bounds__(kJ2Block, 2)
fb_join2_probe_kernel(const uint64_t* __restrict__ pkeys, const uint8_t* __restrict__ pvalid, int64_t nprobe_all,
                      const uint64_t* __restrict__ bkeys, const uint32_t* __restrict__ table, int64_t capacity,
                      FbDiv dv, int64_t region_shift, int outer, uint32_t* __restrict__ cnt,
                      uint32_t* __restrict__ first, int64_t* __restrict__ tile_sums,
                      const int64_t* __restrict__ status, const int64_t* __restrict__ probe_part_off, int p0,
                      int p1) {
  // probe_part_off != nullptr: only the probe rows of hash partitions [p0, p1) (launched right after the
  // build of the same regions, while table and build keys are still in L2); tile totals are then
  // computed afterwards by fb_join2_tile_sums_kernel
  __shared__ int64_t s_warp[kJ2Block / 32];
  const bool unique = status[1] == 0;  // no duplicate build keys: a chain ends at its first match
  const int64_t row_lo = probe_part_off != nullptr ? probe_part_off[p0] : 0;
  const int64_t nprobe = probe_part_off != nullptr ? probe_part_off[p1] : nprobe_all;
  const int64_t ntiles = (nprobe - row_lo + kJ2Tile - 1) / kJ2Tile;
  pkeys += row_lo;
  if (pvalid != nullptr) pvalid += row_lo;
  cnt += row_lo;
  first += row_lo;
  const int64_t nprobe_rel = nprobe - row_lo;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    // the dependent loads of one row (slot -> build key) are latency-bound: keep the first step of all 8
    // rows of this thread in flight together, then finish the (rarer) longer chains row by row
    uint64_t key[kJ2Items];
    uint32_t reg[kJ2Items], off[kJ2Items], e[kJ2Items];  // region id, slot inside the region, slot content
    const int64_t mask = region_shift >= 0 ? (((int64_t)1 << region_shift) - 1) : capacity - 1;
    const int rsh = region_shift >= 0 ? (int)region_shift : 0;
#pragma unroll
    for (int k = 0; k < kJ2Items; ++k) {
      const int64_t i = tile * kJ2Tile + (int64_t)k * kJ2Block + threadIdx.x;
      const bool live = i < nprobe_rel && (pvalid == nullptr || pvalid[i] != 0);
      key[k] = live ? pkeys[i] : 0;
      e[k] = live ? 1u : 0u;
    }
#pragma unroll
    for (int k = 0; k < kJ2Items; ++k) {
      const uint64_t h = fb_hash_single_u64(key[k]);
      reg[k] = region_shift >= 0 ? fb_fastmod(h, dv) : 0u;
      off[k] = (uint32_t)((h >> 10) & (uint64_t)mask);
      if (e[k] != 0) e[k] = __ldg(table + ((int64_t)reg[k] << rsh) + off[k]);
    }
    uint64_t bk[kJ2Items];
#pragma unroll
    for (int k = 0; k < kJ2Items; ++k) bk[k] = e[k] != 0 ? __ldg((const unsigned long long*)bkeys + (e[k] - 1)) : 0;
    int64_t sum = 0;
#pragma unroll
    for (int k = 0; k < kJ2Items; ++k) {
      const int64_t i = tile * kJ2Tile + (int64_t)k * kJ2Block + threadIdx.x;
      if (i >= nprobe_rel) continue;
      uint32_t c = 0, f = kJ2None;
      uint32_t ee = e[k];
      uint64_t bb = bk[k];
      uint32_t ss = off[k];
      const uint32_t* __restrict__ tb = table + ((int64_t)reg[k] << rsh);
      for (int64_t probe = 0; ee != 0 && probe <= mask; ++probe) {
        if (bb == key[k]) {
          if (c == 0) f = ee - 1;
          ++c;
          if (unique) break;
        }
        ss = (uint32_t)((ss + 1) & (uint32_t)mask);
        ee = __ldg(tb + ss);
        if (ee != 0) bb = __ldg((const unsigned long long*)bkeys + (ee - 1));
      }
      if (outer && c == 0) c = 1;  // one NULL-extended row (first stays NONE)
      cnt[i] = c;
      first[i] = f;
      sum += c;
    }
    int64_t total;
    block_exclusive_scan(sum, s_warp, total);
    if (threadIdx.x == 0 && tile_sums != nullptr) tile_sums[tile] = total;
    __syncthreads();
  }
}

// per-tile totals of cnt (pass A run in batches of partitions cannot produce them: its ranges are not tile-aligned)
__global__ void __launch_bounds__(kJ2Block)
fb_join2_tile_sums_kernel(const uint32_t* __restrict__ cnt, int64_t nprobe, int64_t* __restrict__ tile_sums) {
  __shared__ int64_t s_warp[kJ2Block / 32];
  const int64_t ntiles = (nprobe + kJ2Tile - 1) / kJ2Tile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int64_t sum = 0;
#pragma unroll
    for (int k = 0; k < kJ2Items; ++k) {
      const int64_t i = tile * kJ2Tile + (int64_t)k * kJ2Block + threadIdx.x;
      if (i < nprobe) sum += cnt[i];
    }
    int64_t total;
    block_exclusive_scan(sum, s_warp, total);
    if (threadIdx.x == 0) tile_sums[tile] = total;
    __syncthreads();
  }
}

constexpr int kJ2U = 4;  // output rows per thread and step in pass B

// dst[to0 + u * kJ2Block] = has[u] ? src[from[u]] : 0 for the live rows u: all loads first, then all stores
template <typename T>
__device__ __forceinline__ void j2_copy_rows_t(const void* src, void* dst, const int64_t (&from)[kJ2U], int64_t to0,
                                               const bool (&live)[kJ2U], const bool (&has)[kJ2U]) {
  T v[kJ2U];
#pragma unroll
  for (int u = 0; u < kJ2U; ++u) v[u] = (live[u] && has[u]) ? ((const T*)src)[from[u]] : (T)0;
#pragma unroll
  for (int u = 0; u < kJ2U; ++u)
    if (live[u]) ((T*)dst)[to0 + (int64_t)u * kJ2Block] = v[u];
}

__device__ __forceinline__ void j2_copy_rows(const void* src, void* dst, int w, const int64_t (&from)[kJ2U], int64_t to0,
                                             const bool (&live)[kJ2U], const bool (&has)[kJ2U]) {
  switch (w) {
    case 8: j2_copy_rows_t<uint64_t>(src, dst, from, to0, live, has); break;
    case 4: j2_copy_rows_t<uint32_t>(src, dst, from, to0, live, has); break;
    case 2: j2_copy_rows_t<uint16_t>(src, dst, from, to0, live, has); break;
    default: j2_copy_rows_t<uint8_t>(src, dst, from, to0, live, has); break;
  }
}

// pass B
__global__ void __launch_bounds__(kJ2Block, 2)
fb_join2_emit_kernel(const uint64_t* __restrict__ pkeys, int64_t nprobe, const uint64_t* __restrict__ bkeys,
                     const uint32_t* __restrict__ table, int64_t capacity, FbDiv dv, int64_t region_shift,
                     const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ first,
                     const int64_t* __restrict__ tile_base, const __grid_constant__ J2Cols lcols,
                     const __grid_constant__ J2Cols rcols) {
  // output slot of the current window -> (row of the tile, build row): filled by the thread that OWNS the
  // probe row (it walks a chain with duplicates once, resuming across windows), consumed one thread per slot
  __shared__ uint16_t s_slot_row[kJ2Tile];
  __shared__ uint32_t s_slot_b[kJ2Tile];
  __shared__ int64_t s_warp[kJ2Block / 32];
  const int64_t ntiles = (nprobe + kJ2Tile - 1) / kJ2Tile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * kJ2Tile;
    // thread t owns rows [t * 8, t * 8 + 8) of the tile (32 contiguous bytes of cnt / first)
    uint32_t c[kJ2Items], f[kJ2Items];
    int64_t mine = 0;
#pragma unroll
    for (int k = 0; k < kJ2Items; ++k) {
      const int64_t g = row0 + (int64_t)threadIdx.x * kJ2Items + k;
      c[k] = g < nprobe ? cnt[g] : 0;
      f[k] = g < nprobe ? first[g] : kJ2None;
      mine += c[k];
    }
    int64_t total;
    const int64_t my_start = block_exclusive_scan(mine, s_warp, total);
    const int64_t gbase = tile_base[tile];
    // resume state of the (at most one at a time) row with duplicates that this thread is walking
    int walk_k = -1;
    int64_t walk_base = 0, walk_s = 0, walk_mask = 0;
    uint32_t walk_done = 0;
    for (int64_t w0 = 0; w0 < total; w0 += kJ2Tile) {
      const int64_t w1 = w0 + kJ2Tile;
      int64_t o = my_start;
#pragma unroll
      for (int k = 0; k < kJ2Items; ++k) {
        const int64_t lo = o > w0 ? o : w0;
        const int64_t hi = o + c[k] < w1 ? o + c[k] : w1;
        if (lo < hi) {
          const uint16_t r = (uint16_t)(threadIdx.x * kJ2Items + k);
          if (c[k] == 1) {  // unique match (or the NULL-extended row of an outer join)
            s_slot_row[lo - w0] = r;
            s_slot_b[lo - w0] = f[k];
          } else {
            // duplicates of the build key: emit matches number [lo - o, hi - o) of the chain
            const uint64_t key = pkeys[row0 + r];
            if (walk_k != k) {
              walk_k = k;
              walk_done = 0;
              j2_locate(key, dv, region_shift, capacity, walk_base, walk_s, walk_mask);
            }
            int64_t j = lo;
            while (j < hi) {
              const uint32_t e = __ldg(table + walk_base + walk_s);
              walk_s = (walk_s + 1) & walk_mask;
              if (e == 0) break;  // cannot happen: cnt matches exist
              if (__ldg((const unsigned long long*)bkeys + (e - 1)) == key) {
                if ((int64_t)walk_done >= lo - o) {
                  s_slot_row[j - w0] = r;
                  s_slot_b[j - w0] = e - 1;
                  ++j;
                }
                ++walk_done;
              }
            }
          }
        }
        o += c[k];
      }
      __syncthreads();
      const int64_t wn = total - w0 < kJ2Tile ? total - w0 : kJ2Tile;
      // one thread per OUTPUT row, four rows per step: the loads of the four rows are issued together (the
      // column pointers may alias as far as the compiler knows, so row-by-row code would serialise every load
      // behind the previous row's stores)
      for (int64_t j0 = threadIdx.x; j0 < wn; j0 += (int64_t)kJ2Block * kJ2U) {
        int64_t grow[kJ2U], brow[kJ2U];
        bool live[kJ2U], has[kJ2U];
#pragma unroll
        for (int u = 0; u < kJ2U; ++u) {
          const int64_t j = j0 + (int64_t)u * kJ2Block;
          live[u] = j < wn;
          const uint32_t b = live[u] ? s_slot_b[j] : kJ2None;
          grow[u] = row0 + (live[u] ? s_slot_row[j] : 0);
          has[u] = b != kJ2None;
          brow[u] = has[u] ? (int64_t)b : 0;
        }
        const int64_t out0 = gbase + w0 + j0;
        for (int cI = 0; cI < lcols.n; ++cI) j2_copy_rows(lcols.src[cI], lcols.dst[cI], lcols.width[cI], grow, out0, live, live);
        for (int cI = 0; cI < rcols.n; ++cI) {
          j2_copy_rows(rcols.src[cI], rcols.dst[cI], rcols.width[cI], brow, out0, live, has);
          if (rcols.vdst[cI] != nullptr) {
            uint8_t vv[kJ2U];
#pragma unroll
            for (int u = 0; u < kJ2U; ++u)
              vv[u] = has[u] ? (rcols.vsrc[cI] != nullptr ? rcols.vsrc[cI][brow[u]] : (uint8_t)1) : (uint8_t)0;
#pragma unroll
            for (int u = 0; u < kJ2U; ++u)
              if (live[u]) rcols.vdst[cI][out0 + (int64_t)u * kJ2Block] = vv[u];
          }
        }
      }
      __syncthreads();
    }
  }
}

// the checks and the launch shared by fb_range_join_count and fb_range_join_emit
template <bool kEmit>
int range_join_launch(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                      const uint64_t* d_left_codes, const uint8_t* d_left_valid, int64_t nright,
                      const uint64_t* d_start_codes, const int64_t* d_end_keys, const void* d_tree,
                      size_t tree_bytes, const int64_t* d_right_rows, int closed, int outer, int64_t* d_counts,
                      const int64_t* d_offsets, int64_t* d_out_left, int64_t* d_out_right) {
  FB_CHECK(nleft >= 0 && nright >= 0, "negative count");
  FB_CHECK((closed & ~(FB_RANGE_CLOSED_LEFT | FB_RANGE_CLOSED_RIGHT)) == 0, "unknown closed flags %d", closed);
  if (nleft == 0) return 0;
  FB_CHECK(d_run != nullptr && d_run_offsets != nullptr && d_left_codes != nullptr && d_counts != nullptr,
           "NULL run, offsets, codes or counts");
  FB_CHECK(nright == 0 || (d_start_codes != nullptr && d_end_keys != nullptr), "NULL start or end codes");
  const size_t need = fb_window_bounded_scratch_bytes(nright, 1);
  FB_CHECK(need == 0 || (d_tree != nullptr && tree_bytes >= need), "tree too small: %zu < %zu", tree_bytes, need);
  FB_CHECK(!kEmit || (d_right_rows != nullptr && d_offsets != nullptr && d_out_left != nullptr &&
                      d_out_right != nullptr), "NULL rows, offsets or outputs");
  const int64_t grid = (nleft + 255) / 256;
  FB_CHECK(grid < (1LL << 31), "too many rows");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  const RangeTree T{d_end_keys, (const int64_t*)d_tree};
  fb_range_join_kernel<kEmit><<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(
      nleft, d_run, d_run_offsets, d_left_codes, d_left_valid, d_start_codes, T, tree_levels(nright), d_right_rows,
      closed, outer ? 1 : 0, d_counts, d_offsets, d_out_left, d_out_right);
  FB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

size_t fb_join_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * sizeof(Slot) : 0; }

int fb_join_build_u64(int dev, void* stream, int64_t nbuild, const void* keys, const uint8_t* key_valid,
                      int64_t capacity, uint32_t num_parts, void* table, int64_t* d_status,
                      const int64_t* d_part_offsets) {
  FB_CHECK(nbuild >= 0, "nbuild < 0");
  FB_CHECK(capacity >= 2 && (capacity & (capacity - 1)) == 0, "capacity must be a power of two >= 2");
  FB_CHECK(capacity > nbuild, "capacity must exceed the number of build rows");
  FB_CHECK(table != nullptr && d_status != nullptr, "table/status is NULL");
  FB_CHECK(num_parts <= 1 || ((num_parts & (num_parts - 1)) == 0 && (int64_t)num_parts * 2 <= capacity),
           "num_parts must be a power of two <= capacity / 2");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  const FbDiv dv = fb_make_div(num_parts > 1 ? num_parts : 1);
  const int64_t rs = region_shift_of(capacity, num_parts);
  if (num_parts > 1 && d_part_offsets != nullptr && nbuild > 0) {
    // clear + fill a few regions at a time, so that they are still in L2 when the inserts arrive
    // (a table cleared as a whole is back in HBM by then: one random DRAM
    // sector read + write-back per insert)
    const int64_t region_bytes = ((int64_t)1 << rs) * (int64_t)sizeof(Slot);
    int64_t per = l2_batch_bytes() / region_bytes;
    if (per < 1) per = 1;
    FB_CUDA(cudaMemsetAsync(d_status, 0, 4 * sizeof(int64_t), st));
    for (int64_t p0 = 0; p0 < (int64_t)num_parts; p0 += per) {
      const int64_t p1 = p0 + per < (int64_t)num_parts ? p0 + per : (int64_t)num_parts;
      const int64_t nslots = (p1 - p0) << rs;
      fb_join_clear_kernel<<<grid_for(dev, nslots / 4 + 1), 256, 0, st>>>((Slot*)table, p0 << rs, nslots, nullptr);
      const int64_t est = nbuild / num_parts * (p1 - p0) * 5 / 4 + 256;
      fb_join_build_kernel<<<grid_for(dev, est), 256, 0, st>>>((const uint64_t*)keys, key_valid, nbuild, (Slot*)table,
                                                              capacity, d_status, dv, rs, d_part_offsets, (int)p0,
                                                              (int)p1);
    }
    FB_CUDA(cudaGetLastError());
    return 0;
  }
  fb_join_clear_kernel<<<grid_for(dev, capacity), 256, 0, st>>>((Slot*)table, 0, capacity, d_status);
  FB_CUDA(cudaGetLastError());
  if (nbuild > 0) {
    fb_join_build_kernel<<<grid_for(dev, nbuild), 256, 0, st>>>((const uint64_t*)keys, key_valid, nbuild,
                                                                (Slot*)table, capacity, d_status, dv, rs, nullptr, 0, 0);
    FB_CUDA(cudaGetLastError());
  }
  return 0;
}

int fb_join_probe_count_u64(int dev, void* stream, int64_t nprobe, const void* keys,
                            const uint8_t* key_valid, int64_t capacity, uint32_t num_parts,
                            const void* table, int outer, int64_t* out_counts, int64_t* out_first) {
  FB_CHECK(nprobe >= 0, "nprobe < 0");
  if (nprobe == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_join_probe_kernel<false><<<grid_for(dev, nprobe), 256, 0, (cudaStream_t)stream>>>(
      (const uint64_t*)keys, key_valid, nprobe, (const Slot*)table, capacity, outer, out_counts, nullptr,
      nullptr, nullptr, fb_make_div(num_parts > 1 ? num_parts : 1), region_shift_of(capacity, num_parts),
      out_first);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_join_probe_write_u64(int dev, void* stream, int64_t nprobe, const void* keys,
                            const uint8_t* key_valid, int64_t capacity, uint32_t num_parts,
                            const void* table, int outer, const int64_t* offsets, int64_t* out_probe_idx,
                            int64_t* out_build_idx, const int64_t* counts, const int64_t* first) {
  FB_CHECK(nprobe >= 0, "nprobe < 0");
  if (nprobe == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_join_probe_kernel<true><<<grid_for(dev, nprobe), 256, 0, (cudaStream_t)stream>>>(
      (const uint64_t*)keys, key_valid, nprobe, (const Slot*)table, capacity, outer,
      (counts != nullptr && first != nullptr) ? (int64_t*)counts : nullptr, offsets, out_probe_idx, out_build_idx,
      fb_make_div(num_parts > 1 ? num_parts : 1), region_shift_of(capacity, num_parts),
      (counts != nullptr && first != nullptr) ? (int64_t*)first : nullptr);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_join_mark_matched(int dev, void* stream, const int64_t* build_idx, int64_t n, uint8_t* matched) {
  if (n <= 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_join_mark_kernel<<<grid_for(dev, n), 256, 0, (cudaStream_t)stream>>>(build_idx, n, matched);
  FB_CUDA(cudaGetLastError());
  return 0;
}

size_t fb_exclusive_scan_scratch_bytes(int64_t n) {
  int64_t ntiles = (n + kScanTile - 1) / kScanTile;
  return (size_t)(ntiles + 1) * sizeof(int64_t);
}

int fb_exclusive_scan_i64(int dev, void* stream, int64_t n, const int64_t* in, int64_t* out,
                          int64_t* out_total, void* scratch, size_t scratch_bytes) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(out_total != nullptr, "out_total is NULL");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    FB_CUDA(cudaMemsetAsync(out_total, 0, sizeof(int64_t), st));
    return 0;
  }
  FB_CHECK(scratch != nullptr && scratch_bytes >= fb_exclusive_scan_scratch_bytes(n), "scan scratch too small");
  const int64_t ntiles = (n + kScanTile - 1) / kScanTile;
  int64_t* sums = (int64_t*)scratch;
  fb_scan_tile_sums_kernel<<<(unsigned)ntiles, kScanBlock, 0, st>>>(in, n, sums);
  FB_CUDA(cudaGetLastError());
  fb_scan_sums_kernel<<<1, kScanBlock, 0, st>>>(sums, ntiles, out_total);
  FB_CUDA(cudaGetLastError());
  fb_scan_tiles_kernel<<<(unsigned)ntiles, kScanBlock, 0, st>>>(in, n, sums, out);
  FB_CUDA(cudaGetLastError());
  return 0;
}

size_t fb_compact_scratch_bytes(int64_t n) { return fb_exclusive_scan_scratch_bytes(n); }

int fb_compact_indices(int dev, void* stream, const uint8_t* mask, int64_t n, int64_t* out_idx,
                       int64_t* d_count, void* scratch, size_t scratch_bytes) {
  FB_CHECK(n >= 0 && d_count != nullptr, "bad arguments");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    FB_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int64_t), st));
    return 0;
  }
  FB_CHECK(scratch != nullptr && scratch_bytes >= fb_compact_scratch_bytes(n), "compaction scratch too small");
  const int64_t ntiles = (n + kScanTile - 1) / kScanTile;
  int64_t* counts = (int64_t*)scratch;
  fb_mask_tile_counts_kernel<<<(unsigned)ntiles, kScanBlock, 0, st>>>(mask, n, counts);
  FB_CUDA(cudaGetLastError());
  fb_scan_sums_kernel<<<1, kScanBlock, 0, st>>>(counts, ntiles, d_count);
  FB_CUDA(cudaGetLastError());
  fb_mask_write_kernel<<<(unsigned)ntiles, kScanBlock, 0, st>>>(mask, n, counts, out_idx);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_gather_rows(int dev, void* stream, int ncols, const void* const* d_src_cols, void* const* d_dst_cols,
                   const int32_t* d_widths, const uint8_t* const* d_src_valid, uint8_t* const* d_dst_valid,
                   const int64_t* idx, int64_t n) {
  FB_CHECK(ncols >= 0 && n >= 0, "negative count");
  if (ncols == 0 || n == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  dim3 grid(grid_for(dev, n, 4), (unsigned)ncols);
  fb_gather_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_src_cols, d_dst_cols, d_widths, d_src_valid,
                                                               d_dst_valid, idx, n);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_scatter_rows(int dev, void* stream, int ncols, const void* const* d_src_cols, void* const* d_dst_cols,
                    const int32_t* d_widths, const uint8_t* const* d_src_valid, uint8_t* const* d_dst_valid,
                    const int64_t* idx, int64_t n) {
  FB_CHECK(ncols >= 0 && n >= 0, "negative count");
  if (ncols == 0 || n == 0) return 0;
  FB_CHECK(d_src_valid != nullptr && d_dst_valid != nullptr, "validity pointer tables are NULL");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_scatter_rows_kernel<<<grid_for(dev, n, 4), 256, 0, (cudaStream_t)stream>>>(
      d_src_cols, d_dst_cols, d_widths, d_src_valid, d_dst_valid, idx, n, ncols);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_asof_search(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                   const uint64_t* d_left_codes, const uint8_t* d_left_valid, const uint64_t* d_right_codes,
                   const int64_t* d_right_rows, int key_class, int direction, int allow_exact_matches,
                   int has_tolerance, uint64_t tolerance, int64_t* d_out) {
  FB_CHECK(nleft >= 0, "negative count");
  FB_CHECK(key_class == FB_RANGE_KEY_I64 || key_class == FB_RANGE_KEY_U64 || key_class == FB_RANGE_KEY_F64,
           "unknown key class %d", key_class);
  FB_CHECK(direction == FB_ASOF_BACKWARD || direction == FB_ASOF_FORWARD || direction == FB_ASOF_NEAREST,
           "unknown direction %d", direction);
  if (nleft == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_asof_search_kernel<<<(unsigned)((nleft + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      nleft, d_run, d_run_offsets, d_left_codes, d_left_valid, d_right_codes, d_right_rows, key_class, direction,
      allow_exact_matches ? 0 : 1, has_tolerance ? 1 : 0, tolerance, d_out);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_range_join_count(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                        const uint64_t* d_left_codes, const uint8_t* d_left_valid, int64_t nright,
                        const uint64_t* d_start_codes, const int64_t* d_end_keys, const void* d_tree,
                        size_t tree_bytes, int closed, int outer, int64_t* d_counts) {
  return range_join_launch<false>(dev, stream, nleft, d_run, d_run_offsets, d_left_codes, d_left_valid, nright,
                                  d_start_codes, d_end_keys, d_tree, tree_bytes, nullptr, closed, outer, d_counts,
                                  nullptr, nullptr, nullptr);
}

int fb_range_join_emit(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                       const uint64_t* d_left_codes, const uint8_t* d_left_valid, int64_t nright,
                       const uint64_t* d_start_codes, const int64_t* d_end_keys, const void* d_tree,
                       size_t tree_bytes, const int64_t* d_right_rows, int closed, int outer,
                       const int64_t* d_counts, const int64_t* d_offsets, int64_t* d_out_left,
                       int64_t* d_out_right) {
  return range_join_launch<true>(dev, stream, nleft, d_run, d_run_offsets, d_left_codes, d_left_valid, nright,
                                 d_start_codes, d_end_keys, d_tree, tree_bytes, d_right_rows, closed, outer,
                                 (int64_t*)d_counts, d_offsets, d_out_left, d_out_right);
}

// ---- K7 fast path (see the kernels above) ------------------------------------------------------------
size_t fb_join2_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * sizeof(uint32_t) : 0; }

int fb_join2_build(int dev, void* stream, int64_t nbuild, const void* keys, const uint8_t* key_valid,
                   int64_t capacity, uint32_t num_parts, void* table, int64_t* d_status,
                   const int64_t* d_part_offsets) {
  FB_CHECK(nbuild >= 0 && nbuild < (int64_t)0xFFFFFFFF, "nbuild out of range");
  FB_CHECK(capacity >= 4 && (capacity & (capacity - 1)) == 0 && capacity <= ((int64_t)1 << 32),
           "capacity must be a power of two in [4, 2^32]");
  FB_CHECK(capacity > nbuild, "capacity must exceed the number of build rows");
  FB_CHECK(table != nullptr && d_status != nullptr, "table/status is NULL");
  FB_CHECK(num_parts <= 1 || ((num_parts & (num_parts - 1)) == 0 && (int64_t)num_parts * 4 <= capacity),
           "num_parts must be a power of two <= capacity / 4");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  const FbDiv dv = fb_make_div(num_parts > 1 ? num_parts : 1);
  const int64_t rs = region_shift_of(capacity, num_parts);
  FB_CUDA(cudaMemsetAsync(d_status, 0, 4 * sizeof(int64_t), st));
  if (num_parts > 1 && d_part_offsets != nullptr && nbuild > 0) {
    // clear + fill batches of regions that fit L2, so that the inserts hit lines that are still there
    const int64_t region_bytes = ((int64_t)1 << rs) * (int64_t)sizeof(uint32_t);
    int64_t per = ((int64_t)48 << 20) / region_bytes;
    if (per < 1) per = 1;
    for (int64_t p0 = 0; p0 < (int64_t)num_parts; p0 += per) {
      const int64_t p1 = p0 + per < (int64_t)num_parts ? p0 + per : (int64_t)num_parts;
      const int64_t nslots = (p1 - p0) << rs;
      fb_join2_clear_kernel<<<grid_for(dev, nslots / 4 + 1), 256, 0, st>>>((uint32_t*)table, p0 << rs, nslots);
      const int64_t est = nbuild / num_parts * (p1 - p0) * 5 / 4 + 256;
      fb_join2_build_kernel<<<grid_for(dev, est), 256, 0, st>>>((const uint64_t*)keys, key_valid, nbuild,
                                                               (uint32_t*)table, capacity, d_status, dv, rs,
                                                               d_part_offsets, (int)p0, (int)p1);
    }
    FB_CUDA(cudaGetLastError());
    return 0;
  }
  fb_join2_clear_kernel<<<grid_for(dev, capacity / 4), 256, 0, st>>>((uint32_t*)table, 0, capacity);
  FB_CUDA(cudaGetLastError());
  if (nbuild > 0) {
    fb_join2_build_kernel<<<grid_for(dev, nbuild), 256, 0, st>>>((const uint64_t*)keys, key_valid, nbuild,
                                                                 (uint32_t*)table, capacity, d_status, dv, rs,
                                                                 nullptr, 0, 0);
    FB_CUDA(cudaGetLastError());
  }
  return 0;
}

size_t fb_join2_tiles_bytes(int64_t nprobe) {
  return (size_t)((nprobe + kJ2Tile - 1) / kJ2Tile + 1) * sizeof(int64_t);
}

int fb_join2_probe(int dev, void* stream, int64_t nprobe, const void* probe_keys, const uint8_t* probe_valid,
                   const void* build_keys, int64_t capacity, uint32_t num_parts, const void* table, int outer,
                   uint32_t* out_cnt, uint32_t* out_first, int64_t* d_tile_base, int64_t* d_total,
                   const int64_t* d_status) {
  FB_CHECK(nprobe >= 0, "nprobe < 0");
  FB_CHECK(d_total != nullptr && d_status != nullptr, "d_total / d_status is NULL");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (nprobe == 0) {
    FB_CUDA(cudaMemsetAsync(d_total, 0, sizeof(int64_t), st));
    return 0;
  }
  const int64_t ntiles = (nprobe + kJ2Tile - 1) / kJ2Tile;
  int64_t grid = ntiles < (int64_t)fb_sm_count(dev) * 4 ? ntiles : (int64_t)fb_sm_count(dev) * 4;
  fb_join2_probe_kernel<<<(unsigned)grid, kJ2Block, 0, st>>>(
      (const uint64_t*)probe_keys, probe_valid, nprobe, (const uint64_t*)build_keys, (const uint32_t*)table,
      capacity, fb_make_div(num_parts > 1 ? num_parts : 1), region_shift_of(capacity, num_parts), outer, out_cnt,
      out_first, d_tile_base, d_status, nullptr, 0, 0);
  FB_CUDA(cudaGetLastError());
  fb_scan_sums_kernel<<<1, kScanBlock, 0, st>>>(d_tile_base, ntiles, d_total);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_join2_build_probe(int dev, void* stream, int64_t nbuild, const void* build_keys, const uint8_t* build_valid,
                         const int64_t* d_build_part_offsets, int64_t nprobe, const void* probe_keys,
                         const uint8_t* probe_valid, const int64_t* d_probe_part_offsets, int64_t capacity,
                         uint32_t num_parts, void* table, int outer, uint32_t* out_cnt, uint32_t* out_first,
                         int64_t* d_tile_base, int64_t* d_total, int64_t* d_status) {
  FB_CHECK(nbuild >= 0 && nbuild < (int64_t)0xFFFFFFFF && nprobe >= 0, "row counts out of range");
  FB_CHECK(capacity >= 4 && (capacity & (capacity - 1)) == 0 && capacity <= ((int64_t)1 << 32),
           "capacity must be a power of two in [4, 2^32]");
  FB_CHECK(capacity > nbuild, "capacity must exceed the number of build rows");
  FB_CHECK(num_parts > 1 && (num_parts & (num_parts - 1)) == 0 && (int64_t)num_parts * 4 <= capacity,
           "num_parts must be a power of two in [2, capacity / 4]");
  FB_CHECK(table != nullptr && d_status != nullptr && d_total != nullptr, "table / status / total is NULL");
  FB_CHECK(d_build_part_offsets != nullptr && d_probe_part_offsets != nullptr, "partition offsets are NULL");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  const FbDiv dv = fb_make_div(num_parts);
  const int64_t rs = region_shift_of(capacity, num_parts);
  FB_CUDA(cudaMemsetAsync(d_status, 0, 4 * sizeof(int64_t), st));
  if (nprobe == 0) {
    FB_CUDA(cudaMemsetAsync(d_total, 0, sizeof(int64_t), st));
    return 0;
  }
  // Batches of regions that fit L2 TOGETHER WITH the build keys of the same partitions: clear, insert, and
  // probe the probe rows of these partitions at once - the probe's two dependent random reads per step
  // (slot, build key) then hit L2 instead of fetching cold 32-byte sectors from HBM.  Both kernels are
  // chains of dependent L2 accesses (ncu: 22 % / 32 % issue-active, long-scoreboard bound), so the probe of
  // batch b runs on a second stream next to the build of batch b + 1 (disjoint regions): two latency-bound
  // kernels fill the machine better than one.
  const int64_t region_bytes = ((int64_t)1 << rs) * (int64_t)sizeof(uint32_t);
  int64_t per = ((int64_t)24 << 20) / region_bytes;
  if (per < 1) per = 1;
  const int sms = fb_sm_count(dev);
  cudaStream_t s2 = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr}, ev_done = nullptr;
  FB_CUDA(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) FB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
  FB_CUDA(cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming));
  int b = 0;
  for (int64_t p0 = 0; p0 < (int64_t)num_parts; p0 += per, ++b) {
    const int64_t p1 = p0 + per < (int64_t)num_parts ? p0 + per : (int64_t)num_parts;
    const int64_t nslots = (p1 - p0) << rs;
    fb_join2_clear_kernel<<<grid_for(dev, nslots / 4 + 1), 256, 0, st>>>((uint32_t*)table, p0 << rs, nslots);
    if (nbuild > 0) {
      const int64_t est = nbuild / num_parts * (p1 - p0) * 5 / 4 + 256;
      fb_join2_build_kernel<<<grid_for(dev, est), 256, 0, st>>>((const uint64_t*)build_keys, build_valid, nbuild,
                                                               (uint32_t*)table, capacity, d_status, dv, rs,
                                                               d_build_part_offsets, (int)p0, (int)p1);
    }
    cudaEventRecord(ev[b & 1], st);
    cudaStreamWaitEvent(s2, ev[b & 1], 0);
    const int64_t est_tiles = (nprobe / num_parts * (p1 - p0) * 5 / 4 + kJ2Tile) / kJ2Tile;
    int64_t grid = est_tiles < (int64_t)sms * 2 ? est_tiles : (int64_t)sms * 2;
    if (grid < 1) grid = 1;
    fb_join2_probe_kernel<<<(unsigned)grid, kJ2Block, 0, s2>>>(
        (const uint64_t*)probe_keys, probe_valid, nprobe, (const uint64_t*)build_keys, (const uint32_t*)table, capacity,
        dv, rs, outer, out_cnt, out_first, nullptr, d_status, d_probe_part_offsets, (int)p0, (int)p1);
  }
  cudaEventRecord(ev_done, s2);
  cudaStreamWaitEvent(st, ev_done, 0);
  const cudaError_t launch_err = cudaGetLastError();
  cudaEventDestroy(ev[0]);
  cudaEventDestroy(ev[1]);
  cudaEventDestroy(ev_done);
  cudaStreamDestroy(s2);  // released once its work has completed
  FB_CUDA(launch_err);
  const int64_t ntiles = (nprobe + kJ2Tile - 1) / kJ2Tile;
  int64_t grid = ntiles < (int64_t)sms * 4 ? ntiles : (int64_t)sms * 4;
  fb_join2_tile_sums_kernel<<<(unsigned)grid, kJ2Block, 0, st>>>(out_cnt, nprobe, d_tile_base);
  fb_scan_sums_kernel<<<1, kScanBlock, 0, st>>>(d_tile_base, ntiles, d_total);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_join2_emit(int dev, void* stream, int64_t nprobe, const void* probe_keys, const void* build_keys,
                  int64_t capacity, uint32_t num_parts, const void* table, const uint32_t* cnt,
                  const uint32_t* first, const int64_t* d_tile_base, int nleft, const void* const* left_src,
                  void* const* left_dst, const int32_t* left_widths, int nright, const void* const* right_src,
                  void* const* right_dst, const int32_t* right_widths, const uint8_t* const* right_valid_src,
                  uint8_t* const* right_valid_dst) {
  FB_CHECK(nprobe >= 0 && nleft >= 0 && nright >= 0, "negative count");
  FB_CHECK(nleft <= kJ2MaxCols && nright <= kJ2MaxCols, "at most %d columns per side", kJ2MaxCols);
  if (nprobe == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  J2Cols lc, rc;
  memset(&lc, 0, sizeof(lc));
  memset(&rc, 0, sizeof(rc));
  lc.n = nleft;
  rc.n = nright;
  for (int c = 0; c < nleft; ++c) {
    const int w = left_widths[c];
    FB_CHECK(w == 1 || w == 2 || w == 4 || w == 8, "left column %d has unsupported width %d", c, w);
    lc.src[c] = left_src[c]; lc.dst[c] = left_dst[c]; lc.width[c] = w;
  }
  for (int c = 0; c < nright; ++c) {
    const int w = right_widths[c];
    FB_CHECK(w == 1 || w == 2 || w == 4 || w == 8, "right column %d has unsupported width %d", c, w);
    rc.src[c] = right_src[c]; rc.dst[c] = right_dst[c]; rc.width[c] = w;
    rc.vsrc[c] = right_valid_src ? right_valid_src[c] : nullptr;
    rc.vdst[c] = right_valid_dst ? right_valid_dst[c] : nullptr;
  }
  const int64_t ntiles = (nprobe + kJ2Tile - 1) / kJ2Tile;
  int64_t grid = ntiles < (int64_t)fb_sm_count(dev) * 4 ? ntiles : (int64_t)fb_sm_count(dev) * 4;
  fb_join2_emit_kernel<<<(unsigned)grid, kJ2Block, 0, (cudaStream_t)stream>>>(
      (const uint64_t*)probe_keys, nprobe, (const uint64_t*)build_keys, (const uint32_t*)table, capacity,
      fb_make_div(num_parts > 1 ? num_parts : 1), region_shift_of(capacity, num_parts), cnt, first, d_tile_base, lc,
      rc);
  FB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
