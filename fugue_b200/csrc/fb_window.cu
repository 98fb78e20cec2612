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
//
// Moving frames (ROWS BETWEEN start AND end, fb_window_frame) use van Herk / Gil-Werman: rows are cut
// into blocks of W = end - start + 1 rows aligned to multiples of W, and two scans restart at every
// block as well as every segment bound: P[i], op from the later of (block start, segment start) to i, and
// S[i], op from i to the earlier of (block end, segment end).  A frame [lo, hi] clipped to its segment
// holds at most W rows, so it lies in at most two blocks: it is S[lo] (+) P[hi] when it crosses a block
// bound, else P[hi] when lo is where P[hi]'s run starts, else S[lo] (hi is then where S[lo]'s run ends).
// O(1) per row for every op, exact for MIN / MAX, and every f64 sum adds frame values only.
//   - W <= FB_FRAME_TILE_MAX_WIDTH: one launch; a CTA stages its rows plus the W - 1 halo in shared
//     memory, scans P and S there and writes each output once (inputs read 1 + (W - 1) / tile times).
//   - otherwise, and with an unbounded side: P and S by the three-launch scan above (block heads added,
//     S walking rows in reverse) into scratch, then a combine launch.  (None, e) is P without blocks read
//     at hi; (s, None) is S without blocks read at lo.
//
// Value frames (RANGE BETWEEN) have a different width on every row, so they take two other kernels:
//   - fb_window_range_bounds: per row, [lo, hi] by a galloping lower_bound / upper_bound from the row over
//     its segment's non-NULL run (the NULL keys are the segment's tail), in the order-key domain of the sort.
//   - fb_window_bounded: the op over any [lo, hi] from an aligned power-of-two block tree.  Level l holds op
//     and count of rows [m 2^l, (m + 1) 2^l), built pairwise level by level; an interval is at most two
//     blocks per level (the canonical decomposition of a bottom-up segment tree), combined left to right.
//     Blocks ignore segments: a frame never crosses its segment and its blocks lie inside it.  The counts
//     live in the tree beside the values because the combination needs them anyway (a block without a
//     valid row takes no part, so MIN / MAX need no identity).
#include <mutex>

#include "fb_common.cuh"
#include "fb_tree.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;                  // consecutive rows per thread
constexpr int kTile = kThreads * kItems;   // rows per CTA

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

// Every scan state is kWords 8-byte words and the flag f, "a segment starts in here".  zip(a, b, g) calls g on each
// word of a with the same word of b, in order (a and b may be one state); shuffles and the tile states in scratch
// go through it.

// (value, count of valid rows, f) of a run of consecutive rows
struct St {
  uint64_t v;
  int64_t c;
  int32_t f;
  static constexpr int kWords = 2;
  template <class A, class B, class G>
  __device__ __forceinline__ static void zip(A& a, B& b, G&& g) { g(a.v, b.v); g(a.c, b.c); }
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

// (count, mean, M2, "a segment starts in here") of the valid values of a run of consecutive rows: the state of
// fb_segmented_moments
struct MSt {
  int64_t c;
  double mean, m2;
  int32_t f;
  static constexpr int kWords = 3;
  template <class A, class B, class G>
  __device__ __forceinline__ static void zip(A& a, B& b, G&& g) { g(a.c, b.c); g(a.mean, b.mean); g(a.m2, b.m2); }
};

// `a` followed by `b`: Chan, Golub & LeVeque's pairwise update; a run without a valid row takes no part
__device__ __forceinline__ MSt combine(int, const MSt& a, const MSt& b) {
  if (b.f) return b;
  if (b.c == 0) return MSt{a.c, a.mean, a.m2, a.f};
  if (a.c == 0) return MSt{b.c, b.mean, b.m2, a.f};
  const int64_t n = a.c + b.c;
  const double delta = b.mean - a.mean;
  const double wb = (double)b.c * __drcp_rn((double)n);  // nb / n within 2 u; a division call spilled
  return MSt{n, a.mean + delta * wb, a.m2 + b.m2 + delta * delta * (double)a.c * wb, a.f};
}

// (count, mean x, mean y, Sxx, Syy, Sxy, "a segment starts in here") of the pair rows of a run of consecutive
// rows: the state of fb_segmented_comoments
struct CSt {
  int64_t c;
  double mx, my, sxx, syy, sxy;
  int32_t f;
  static constexpr int kWords = 6;
  template <class A, class B, class G>
  __device__ __forceinline__ static void zip(A& a, B& b, G&& g) {
    g(a.c, b.c); g(a.mx, b.mx); g(a.my, b.my);
    g(a.sxx, b.sxx); g(a.syy, b.syy); g(a.sxy, b.sxy);
  }
};

// `a` followed by `b`: Chan's pairwise update with the cross term dx * dy * na * nb / n.  A non-finite mean
// difference means a non-finite value (or an overflow): the mean is then the weighted sum of the two, which
// gives +-inf or NaN as the sum of the values would, where the update form would give inf - inf = NaN.
__device__ __forceinline__ CSt combine(int, const CSt& a, const CSt& b) {
  if (b.f) return b;
  if (b.c == 0) return CSt{a.c, a.mx, a.my, a.sxx, a.syy, a.sxy, a.f};
  if (a.c == 0) return CSt{b.c, b.mx, b.my, b.sxx, b.syy, b.sxy, a.f};
  const int64_t n = a.c + b.c;
  const double dx = b.mx - a.mx, dy = b.my - a.my;
  const double rn = __drcp_rn((double)n);
  const double wb = (double)b.c * rn;  // nb / n within 2 u
  const double na = (double)a.c, nb = (double)b.c;
  const double mx = isfinite(dx) ? a.mx + dx * wb : (a.mx * na + b.mx * nb) * rn;
  const double my = isfinite(dy) ? a.my + dy * wb : (a.my * na + b.my * nb) * rn;
  return CSt{n, mx, my, a.sxx + b.sxx + dx * dx * na * wb, a.syy + b.syy + dy * dy * na * wb,
             a.sxy + b.sxy + dx * dy * na * wb, a.f};
}

// (count, mean, M2, M3, M4, "a segment starts in here") of the valid values of a run of consecutive rows: the state
// of fb_segmented_shape_moments
struct SSt {
  int64_t c;
  double mean, m2, m3, m4;
  int32_t f;
  static constexpr int kWords = 5;
  template <class A, class B, class G>
  __device__ __forceinline__ static void zip(A& a, B& b, G&& g) {
    g(a.c, b.c); g(a.mean, b.mean); g(a.m2, b.m2);
    g(a.m3, b.m3); g(a.m4, b.m4);
  }
};

// `a` followed by `b`: Pebay's pairwise update of the third and fourth central sums beside Chan's M2, written in the
// weights wa = na / n, wb = nb / n.  Every right-hand side reads the old sums.  Equal values give delta = 0 exactly,
// so a constant run keeps M2 = M3 = M4 = 0; a run without a valid row takes no part.
__device__ __forceinline__ SSt combine(int, const SSt& a, const SSt& b) {
  if (b.f) return b;
  if (b.c == 0) return SSt{a.c, a.mean, a.m2, a.m3, a.m4, a.f};
  if (a.c == 0) return SSt{b.c, b.mean, b.m2, b.m3, b.m4, a.f};
  const int64_t n = a.c + b.c;
  const double rn = __drcp_rn((double)n);
  const double wa = (double)a.c * rn, wb = (double)b.c * rn;  // na / n, nb / n within 2 u
  const double d = b.mean - a.mean;
  const double d2 = d * d;
  const double t2 = d2 * (double)a.c * wb;  // d^2 na nb / n
  return SSt{n, a.mean + d * wb, a.m2 + b.m2 + t2,
             a.m3 + b.m3 + t2 * d * (wa - wb) + 3.0 * d * (wa * b.m2 - wb * a.m2),
             a.m4 + b.m4 + t2 * d2 * (wa * wa - wa * wb + wb * wb) + 6.0 * d2 * (wa * wa * b.m2 + wb * wb * a.m2) +
                 4.0 * d * (wa * b.m3 - wb * a.m3),
             a.f};
}

// ---- exponentially weighted moments (fb_segmented_ewm) ----
// A column's decay over a position difference dt (int64, exact): beta^dt = exp2(k dt), k = log2(1 - alpha) when the
// positions are row indices or observation ordinals (obs), -1 / halflife when they are times.  A new observation weighs
// 1 with adjust, else alpha times the total weight before it.
struct EwOp {
  double k, alpha;
  int32_t adjust, obs;
};
__device__ __forceinline__ bool is_count_op(const EwOp&) { return false; }
__device__ __forceinline__ double decay(const EwOp& op, int64_t dt) { return dt == 0 ? 1.0 : exp2(op.k * (double)dt); }

// The observations of a run of consecutive rows: their count c, the positions t1 and tl of the first and the last, the
// first value x1, q and, over the others, (w, w2, mean, cm): the sums of the weights and of their squares, the weighted
// mean and the sum of w (x - mean)^2, every weight seen from tl.  With adjust the weights are absolute and q is x1's
// own weight (beta^(tl - t1)); the total weight of a run is at least its last observation's 1.  Without adjust every
// weight is a share of the run's total weight at tl (so q + w = 1): q is the share of all that came before the run's
// second observation (x1 and, for a run inside a partition, the rows before the run).  Keeping shares rather than
// pandas' running total T, which shrinks or grows by beta^g + alpha at every gap, is what keeps a long partition
// from overflowing or underflowing (DESIGN §7s).
struct EwSt {
  int64_t c, t1, tl;
  double x1, q, w, w2, mean, cm;
  int32_t f;
  static constexpr int kWords = 9;
  template <class A, class B, class G>
  __device__ __forceinline__ static void zip(A& a, B& b, G&& g) {
    g(a.c, b.c); g(a.t1, b.t1); g(a.tl, b.tl); g(a.x1, b.x1); g(a.q, b.q);
    g(a.w, b.w); g(a.w2, b.w2); g(a.mean, b.mean); g(a.cm, b.cm);
  }
};

// (sum of weights, of squared weights, weighted mean, sum of w (x - mean)^2) of a weighted set
struct EwSum {
  double w, w2, mean, cm;
};

// `a` followed by `b`: the weighted Chan update.  A non-finite mean difference means a non-finite value: the mean is
// then the weighted sum of the two, as in CSt's combine.  A weight decayed to 0 (alpha = 1, or an underflow) leaves
// nothing of `a` but its sums, so that 0 / 0 never occurs.  The weights divide, not multiply by a reciprocal: a total
// weight decayed below 2^-1022 has no finite reciprocal.
__device__ __forceinline__ EwSum ew_merge(const EwSum& a, const EwSum& b) {
  if (a.w == 0.0) return EwSum{b.w, a.w2 + b.w2, b.mean, a.cm + b.cm};
  const double w = a.w + b.w;
  const double d = b.mean - a.mean;
  const double wb = b.w / w;
  return EwSum{w, a.w2 + b.w2, isfinite(d) ? a.mean + d * wb : (a.mean * a.w + b.mean * b.w) / w,
               a.cm + b.cm + d * d * a.w * wb};
}

// a run's first observation (weight q) merged with its others: the sums of the run from its partition's first
// observation on, when the run holds it
__device__ __forceinline__ EwSum ew_total(const EwSt& s) {
  const EwSum p{s.q, s.q * s.q, s.x1, s.x1 - s.x1};
  return s.c > 1 ? ew_merge(p, EwSum{s.w, s.w2, s.mean, s.cm}) : p;
}

// `a` followed by `b`: a's others (scaled by fa), b's first observation (weight w1) and b's others merge in that order,
// and everything a held up to its second observation keeps the share a.q fa.  With adjust, fa = beta^(b.tl - a.tl) and
// w1 = b.q.  Without adjust, a's total (1 at a.tl) decays to beta^g at b's first observation, which then weighs alpha:
// a keeps beta^g / (beta^g + alpha) and b's first observation alpha / (beta^g + alpha) of the total there, and b.q of
// that total is what is left of it at b.tl; b's others are already shares of the total at b.tl.  A run without an
// observation takes no part.
__device__ __forceinline__ EwSt combine(const EwOp& op, const EwSt& a, const EwSt& b) {
  if (b.f) return b;
  if (b.c == 0) return a;
  if (a.c == 0) return EwSt{b.c, b.t1, b.tl, b.x1, b.q, b.w, b.w2, b.mean, b.cm, a.f};
  double fa, w1;
  if (op.adjust) {
    fa = decay(op, op.obs ? b.c : b.tl - a.tl);
    w1 = b.q;
  } else {
    const double bg = decay(op, op.obs ? 1 : b.t1 - a.tl);
    const double den = bg + op.alpha;
    fa = b.q * (bg / den);
    w1 = b.q * (op.alpha / den);
  }
  EwSum r{w1, w1 * w1, b.x1, b.x1 - b.x1};
  if (a.c > 1) r = ew_merge(EwSum{a.w * fa, a.w2 * fa * fa, a.mean, a.cm * fa}, r);
  if (b.c > 1) r = ew_merge(r, EwSum{b.w, b.w2, b.mean, b.cm});
  return EwSt{a.c + b.c, a.t1, b.tl, a.x1, a.q * fa, r.w, r.w2, r.mean, r.cm, a.f};
}

template <class S>
__device__ __forceinline__ S shfl_up(const S& s, int d) {
  S r;
  S::zip(r, s, [d](auto& w, const auto& x) { w = __shfl_up_sync(0xFFFFFFFFu, x, d); });
  r.f = __shfl_up_sync(0xFFFFFFFFu, s.f, d);
  return r;
}

template <class S>
__device__ __forceinline__ S shfl_down(const S& s, int d) {
  S r;
  S::zip(r, s, [d](auto& w, const auto& x) { w = __shfl_down_sync(0xFFFFFFFFu, x, d); });
  r.f = __shfl_down_sync(0xFFFFFFFFu, s.f, d);
  return r;
}

// Exclusive scan of one state per thread across the CTA, and the CTA total; fixed combination order.
// kRev: the scan runs from the last thread to the first.  S: St, or MSt / CSt / SSt (op unused), or EwSt (op: EwOp).
template <int kWarps, bool kRev = false, class S = St, class Op = int>
__device__ __forceinline__ S block_exclusive(const Op& op, const S& x, S* warp_tot, S* total) {
  const int lane = kRev ? 31 - (threadIdx.x & 31) : threadIdx.x & 31;
  const int w = kRev ? kWarps - 1 - (int)(threadIdx.x >> 5) : threadIdx.x >> 5;
  S inc = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const S o = kRev ? shfl_down(inc, d) : shfl_up(inc, d);
    if (lane >= d) inc = combine(op, o, inc);
  }
  const S ex = kRev ? shfl_down(inc, 1) : shfl_up(inc, 1);
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  S pre{}, tot{};
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

// smallest multiple of b >= x (x >= 0, b >= 1, both below 2^53) without a 64-bit division call
__device__ __forceinline__ int64_t first_multiple(int64_t x, int64_t b) {
  int64_t q = (int64_t)((double)x * __drcp_rn((double)b));  // within a few units of x / b
  while (q * b < x) ++q;
  while (q > 0 && (q - 1) * b >= x) --q;
  return q * b;
}

// Marks head[p - start] for every position p in [start, end) where a run restarts (see fb_segscan_tile_kernel);
// seg_range is two int64 of shared memory.  The caller synchronises before reading head.
template <bool kReverse, bool kBlocks>
__device__ __forceinline__ void mark_heads(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                                           int64_t start, int64_t end, int64_t block, uint8_t* head,
                                           int64_t* seg_range) {
  // ---- segment heads inside [start, end): offsets[s] for s in [segment of `start`, first offset >= end);
  // reversed, offsets o in [nrows - end + 1, nrows - start] (row o - 1 ends a segment) at position nrows - o
  for (int i = threadIdx.x; i < kTile; i += kThreads) head[i] = 0;
  if (threadIdx.x == 0) {
    if (kReverse) {
      seg_range[0] = upper_bound(offsets, nseg + 1, nrows - end);
      seg_range[1] = upper_bound(offsets, nseg + 1, nrows - start);
    } else {
      const int64_t s0 = upper_bound(offsets, nseg + 1, start) - 1;
      seg_range[0] = s0 < 0 ? 0 : s0;
      seg_range[1] = lower_bound(offsets, nseg + 1, end);
    }
  }
  __syncthreads();
  for (int64_t s = seg_range[0] + threadIdx.x; s < seg_range[1]; s += kThreads) {
    const int64_t o = __ldg(offsets + s);
    const int64_t p = kReverse ? nrows - o : o;
    if (p >= start && p < end) head[p - start] = 1;
  }
  if (kBlocks) {  // multiples m of `block` with position (m, or nrows - m reversed) inside the tile
    const int64_t lo = kReverse ? nrows - end + 1 : start, hi = kReverse ? nrows - start : end - 1;
    for (int64_t m = first_multiple(lo, block) + threadIdx.x * block; m <= hi; m += kThreads * block)
      head[(kReverse ? nrows - m : m) - start] = 1;
  }
}

// ---- the segmented scans: one tile kernel, one carry kernel and one launch sequence over a scan's traits ----
// A scan's traits give its State (with combine, its 8-byte words and the flag f), its Cols, the kInputs input
// columns a tile stages, the state of one row (entry), its kOut output words (out for a staged scan, outs for all
// kOut at once otherwise), the carry CTA size and how pass 3 stores:
//   - kStaged: the one output word and the count go through shared memory, then striped (coalesced) stores;
//   - otherwise a thread stores its kItems consecutive rows straight from registers: several outputs per row do
//     not fit the staging buffers, and the stores of a warp still cover whole lines together.
// kFrames: the scan also runs reversed and restarts at block bounds (P and S of fb_window_frame).

// the columns of an f64 statistics scan: x (and y for pairs) with their validity, the count and up to five words out
struct StatCols {
  const double* in[2][FB_SCAN_MAX_COLS];      // x, y
  const uint8_t* valid[2][FB_SCAN_MAX_COLS];  // of x, of y (NULL: every row valid)
  int64_t* out_count[FB_SCAN_MAX_COLS];
  double* out[5][FB_SCAN_MAX_COLS];
  int32_t ncols;
};

// a column's op (0 for the f64 families), input k, its validity and output word o
__device__ __forceinline__ int col_op(const ScanCols& a, int col) { return a.op[col]; }
__device__ __forceinline__ int col_op(const StatCols&, int) { return 0; }
__device__ __forceinline__ bool is_count_op(int op) { return op == FB_AGG_COUNT; }
__device__ __forceinline__ const uint64_t* col_input(const ScanCols& a, int col, int) {
  return (const uint64_t*)a.vals[col];
}
__device__ __forceinline__ const uint64_t* col_input(const StatCols& a, int col, int k) {
  return (const uint64_t*)a.in[k][col];
}
__device__ __forceinline__ const uint8_t* col_valid(const ScanCols& a, int col, int) { return a.valid[col]; }
__device__ __forceinline__ const uint8_t* col_valid(const StatCols& a, int col, int k) { return a.valid[k][col]; }
__device__ __forceinline__ uint64_t* col_output(const ScanCols& a, int col, int) { return (uint64_t*)a.out_vals[col]; }
__device__ __forceinline__ uint64_t* col_output(const StatCols& a, int col, int o) { return (uint64_t*)a.out[o][col]; }
// the 8-byte word of input `src` at row r
template <class Cols>
__device__ __forceinline__ uint64_t col_load(const Cols&, const uint64_t* src, int64_t r) {
  return __ldg((const unsigned long long*)src + r);
}

__device__ __forceinline__ double f64_of(uint64_t b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ uint64_t f64_bits(double x) { return (uint64_t)__double_as_longlong(x); }

// SUM / MIN / MAX / COUNT (fb_segmented_scan, and P / S of fb_window_frame)
struct OpScan {
  using State = St;
  using Cols = ScanCols;
  static constexpr int kInputs = 1, kOut = 1, kCarryThreads = 1024;
  static constexpr bool kStaged = true, kFrames = true;
  template <class Sm>
  __device__ __forceinline__ static St entry(int op, const Sm& sm, int j) {
    const int c = sm.valid[j];
    return St{c && op != FB_AGG_COUNT ? sm.buf[0][padded(j)] : 0, c, sm.head[j]};
  }
  __device__ __forceinline__ static uint64_t out(int, const St& s, int) { return s.v; }
};

// running count and M2 (fb_segmented_moments)
struct MomentScan {
  using State = MSt;
  using Cols = StatCols;
  static constexpr int kInputs = 1, kOut = 1, kCarryThreads = 1024;
  static constexpr bool kStaged = true, kFrames = false;
  // a valid value x enters as (1, x, x - x), so that a NaN or an infinity makes M2 NaN
  template <class Sm>
  __device__ __forceinline__ static MSt entry(int, const Sm& sm, int j) {
    const int c = sm.valid[j];
    const double x = c ? f64_of(sm.buf[0][padded(j)]) : 0.0;
    return MSt{c, x, x - x, sm.head[j]};
  }
  __device__ __forceinline__ static uint64_t out(int, const MSt& s, int) { return f64_bits(s.m2); }
};

// running count, mean x, mean y, Sxx, Syy and Sxy of the rows where x and y are both valid (fb_segmented_comoments)
struct CoMomentScan {
  using State = CSt;
  using Cols = StatCols;
  // half the threads of the other carry kernels: a CSt is twice an MSt, and 1024 threads leave 64 registers each
  static constexpr int kInputs = 2, kOut = 5, kCarryThreads = 512;
  static constexpr bool kStaged = false, kFrames = false;
  // a pair enters as (1, x, y, z, z, z) with z = (x - x) * (y - y), +0 for finite x and y and NaN otherwise, so
  // that a NaN or an infinity on either side makes all three sums NaN
  template <class Sm>
  __device__ __forceinline__ static CSt entry(int, const Sm& sm, int j) {
    const int c = sm.valid[j];
    const double x = c ? f64_of(sm.buf[0][padded(j)]) : 0.0, y = c ? f64_of(sm.buf[1][padded(j)]) : 0.0;
    const double z = (x - x) * (y - y);
    return CSt{c, x, y, z, z, z, sm.head[j]};
  }
  __device__ __forceinline__ static void outs(int, const CSt& s, uint64_t (&v)[kOut]) {
    v[0] = f64_bits(s.mx); v[1] = f64_bits(s.my); v[2] = f64_bits(s.sxx); v[3] = f64_bits(s.syy); v[4] = f64_bits(s.sxy);
  }
};

// running count, M2, M3 and M4 (fb_segmented_shape_moments)
struct ShapeScan {
  using State = SSt;
  using Cols = StatCols;
  // an SSt is five 8-byte words and a flag, near a CSt, so the carry runs the co-moments carry's 512 threads
  static constexpr int kInputs = 1, kOut = 3, kCarryThreads = 512;
  static constexpr bool kStaged = false, kFrames = false;
  // a valid value x enters as (1, x, z, z, z) with z = x - x, +0 for a finite x and NaN otherwise, so that a NaN or
  // an infinity makes M2, M3 and M4 NaN
  template <class Sm>
  __device__ __forceinline__ static SSt entry(int, const Sm& sm, int j) {
    const int c = sm.valid[j];
    const double x = c ? f64_of(sm.buf[0][padded(j)]) : 0.0;
    const double z = x - x;
    return SSt{c, x, z, z, z, sm.head[j]};
  }
  __device__ __forceinline__ static void outs(int, const SSt& s, uint64_t (&v)[kOut]) {
    v[0] = f64_bits(s.m2); v[1] = f64_bits(s.m3); v[2] = f64_bits(s.m4);
  }
};

// the columns of fb_segmented_ewm: x with its validity, the positions (times, or NULL: the row index), the count and
// the mean, w, w2 and cm of ew_total out
struct EwCols {
  const double* x[FB_SCAN_MAX_COLS];
  const uint8_t* valid[FB_SCAN_MAX_COLS];
  const int64_t* t[FB_SCAN_MAX_COLS];
  int64_t* out_count[FB_SCAN_MAX_COLS];
  double* out[4][FB_SCAN_MAX_COLS];
  EwOp op[FB_SCAN_MAX_COLS];
  int32_t ncols;
};

__device__ __forceinline__ EwOp col_op(const EwCols& a, int col) { return a.op[col]; }
__device__ __forceinline__ const uint64_t* col_input(const EwCols& a, int col, int k) {
  return k == 0 ? (const uint64_t*)a.x[col] : (const uint64_t*)a.t[col];
}
__device__ __forceinline__ const uint8_t* col_valid(const EwCols& a, int col, int k) {
  return k == 0 ? a.valid[col] : nullptr;
}
__device__ __forceinline__ uint64_t* col_output(const EwCols& a, int col, int o) { return (uint64_t*)a.out[o][col]; }
__device__ __forceinline__ uint64_t col_load(const EwCols&, const uint64_t* src, int64_t r) {
  return src != nullptr ? __ldg((const unsigned long long*)src + r) : (uint64_t)r;
}

// running exponentially weighted count, mean, w, w2 and cm (fb_segmented_ewm)
struct EwScan {
  using State = EwSt;
  using Cols = EwCols;
  // an EwSt is nine 8-byte words and a flag; at the co-moments carry's 512 threads the carry kernel does not spill
  static constexpr int kInputs = 2, kOut = 4, kCarryThreads = 512;
  static constexpr bool kStaged = false, kFrames = false;
  // a row is an observation when x is valid and not NaN; it enters as (1, t, t, x, 1, 0, 0, 0, 0)
  template <class Sm>
  __device__ __forceinline__ static EwSt entry(const EwOp&, const Sm& sm, int j) {
    const double x = f64_of(sm.buf[0][padded(j)]);
    const int64_t t = (int64_t)sm.buf[1][padded(j)];
    return EwSt{sm.valid[j] && x == x, t, t, x, 1.0, 0.0, 0.0, 0.0, 0.0, sm.head[j]};
  }
  // the mean, W, W2 and C of ew_total, merged once per row
  __device__ __forceinline__ static void outs(const EwOp&, const EwSt& s, uint64_t (&v)[kOut]) {
    const EwSum r = ew_total(s);
    v[0] = f64_bits(r.mean); v[1] = f64_bits(r.w); v[2] = f64_bits(r.w2); v[3] = f64_bits(r.cm);
  }
};

// A tile's rows in shared memory: buf[0, kInputs) the staged input columns; a kStaged scan writes its output word
// over buf[0] and its count into buf[kInputs] in pass 3.
template <class T>
struct TileSmem {
  uint64_t buf[T::kInputs + (T::kStaged ? 1 : 0)][padded(kTile)];
  uint8_t valid[kTile];  // every input of the row valid
  uint8_t head[kTile];
  typename T::State warp_tot[kThreads / 32];
  int64_t seg_range[2];
};

// The tile states in scratch, a struct of arrays: w[k][i] is word k of state i = column * tiles + tile (one array
// of columns x tiles per word), then f[tile], one flag per tile.
template <class S>
struct TileStates {
  uint64_t* w[S::kWords];
  int32_t* f;
};

template <class S>
TileStates<S> tile_states(void* scratch, int64_t nt) {
  TileStates<S> ts;
  for (int k = 0; k < S::kWords; ++k) ts.w[k] = (uint64_t*)scratch + k * nt;
  ts.f = (int32_t*)((uint64_t*)scratch + S::kWords * nt);
  return ts;
}

template <class S>
__device__ __forceinline__ S load_state(const TileStates<S>& ts, int64_t i, int32_t f) {
  S s;
  int k = 0;
  S::zip(s, s, [&](auto& x, auto&) {
    const uint64_t b = ts.w[k++][i];
    memcpy(&x, &b, 8);
  });
  s.f = f;
  return s;
}

template <class S>
__device__ __forceinline__ void store_state(const TileStates<S>& ts, int64_t i, S s) {
  int k = 0;
  S::zip(s, s, [&](auto& x, auto&) {
    uint64_t b;
    memcpy(&b, &x, 8);
    ts.w[k++][i] = b;
  });
}

// kFinal = false: pass 1 (tile states); true: pass 3 (outputs, from the carries of pass 2).
// The scan runs over positions p; position p is row p, or row nrows - 1 - p when kReverse (then a run
// restarts after every segment's last row).  block > 0 also restarts the runs at every row that is a
// multiple of `block` (kReverse: every row r with r + 1 a multiple of `block`); only with kBlocks, so that the
// plain scan compiles without it.
template <class T, bool kFinal, bool kReverse = false, bool kBlocks = false>
__global__ void __launch_bounds__(kThreads)
fb_segscan_tile_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                       const __grid_constant__ typename T::Cols a, int64_t ntiles,
                       const TileStates<typename T::State> ts, int64_t block) {
  using S = typename T::State;
  __shared__ __align__(16) TileSmem<T> sm;
  const int64_t tile = blockIdx.x;
  const int64_t start = tile * kTile;
  const int64_t end = start + kTile < nrows ? start + kTile : nrows;
  const int nloc = (int)(end - start);
  // row of the tile's position i
  const int64_t row0 = kReverse ? nrows - 1 - start : start;
  auto row = [row0](int i) -> int64_t { return kReverse ? row0 - i : row0 + i; };
  mark_heads<kReverse, kBlocks>(nrows, nseg, offsets, start, end, block, sm.head, sm.seg_range);
  const int j0 = threadIdx.x * kItems;
  for (int col = 0; col < a.ncols; ++col) {
    const auto op = col_op(a, col);
    const uint64_t* src[T::kInputs];
    const uint8_t* vm[T::kInputs];
#pragma unroll
    for (int k = 0; k < T::kInputs; ++k) {
      src[k] = col_input(a, col, k);
      vm[k] = col_valid(a, col, k);
    }
    // striped (coalesced) loads into shared memory; rows past the end are invalid.  They read the tile's first row
    // instead, so that every load stays in bounds and none waits on a branch.  A COUNT scan reads no values.
    const bool is_count = is_count_op(op);
    for (int i = threadIdx.x; i < kTile; i += kThreads) {
      const bool in = i < nloc;
      const int64_t r = row(in ? i : 0);
#pragma unroll
      for (int k = 0; k < T::kInputs; ++k)
        if (!is_count) sm.buf[k][padded(i)] = in ? col_load(a, src[k], r) : 0;
      bool ok = true;
#pragma unroll
      for (int k = 0; k < T::kInputs; ++k) ok = ok && (vm[k] == nullptr || __ldg(vm[k] + r) != 0);
      sm.valid[i] = in ? ok : 0;
    }
    __syncthreads();
    S acc{};
#pragma unroll
    for (int k = 0; k < kItems; ++k) acc = combine(op, acc, T::entry(op, sm, j0 + k));
    S total;
    const S pre = block_exclusive<kThreads / 32, false, S>(op, acc, sm.warp_tot, &total);
    const int64_t t = col * ntiles + tile;
    if (!kFinal) {
      if (threadIdx.x == 0) {
        store_state(ts, t, total);
        if (col == 0) ts.f[tile] = total.f;
      }
      continue;
    }
    S run = combine(op, load_state(ts, t, 0), pre);
    if constexpr (T::kStaged) {
      static_assert(T::kOut == 1, "a staged scan has one output word");
#pragma unroll
      for (int k = 0; k < kItems; ++k) {
        const int j = j0 + k;
        run = combine(op, run, T::entry(op, sm, j));
        sm.buf[0][padded(j)] = run.c > 0 ? T::out(op, run, 0) : 0;  // no valid row yet: 0, not whatever preceded the segment
        sm.buf[T::kInputs][padded(j)] = (uint64_t)run.c;
      }
      __syncthreads();
      uint64_t* __restrict__ ov = col_output(a, col, 0);
      int64_t* __restrict__ oc = a.out_count[col];
      for (int i = threadIdx.x; i < nloc; i += kThreads) {
        if (ov != nullptr) ov[row(i)] = sm.buf[0][padded(i)];
        if (oc != nullptr) oc[row(i)] = (int64_t)sm.buf[T::kInputs][padded(i)];
      }
    } else {
      int64_t* __restrict__ oc = a.out_count[col];
#pragma unroll
      for (int k = 0; k < kItems; ++k) {
        const int j = j0 + k;
        run = combine(op, run, T::entry(op, sm, j));
        if (j >= nloc) continue;
        const bool any = run.c > 0;  // no valid row yet: 0, not whatever preceded the segment
        if (oc != nullptr) oc[row(j)] = run.c;
        uint64_t v[T::kOut];
        T::outs(op, run, v);
#pragma unroll
        for (int o = 0; o < T::kOut; ++o) {
          uint64_t* __restrict__ ov = col_output(a, col, o);
          if (ov != nullptr) ov[row(j)] = any ? v[o] : 0;
        }
      }
    }
    __syncthreads();  // shared buffers are refilled by the next column
  }
}

// pass 2: per column, the exclusive segmented scan of the tile states (in place: state -> carry)
template <class T>
__global__ void __launch_bounds__(T::kCarryThreads, 1)
fb_segscan_carry_kernel(int64_t ntiles, const __grid_constant__ typename T::Cols a,
                        const TileStates<typename T::State> ts) {
  using S = typename T::State;
  __shared__ S warp_tot[T::kCarryThreads / 32];
  const int col = blockIdx.x;
  const auto op = col_op(a, col);
  const int64_t o = (int64_t)col * ntiles;
  const int64_t per = (ntiles + T::kCarryThreads - 1) / T::kCarryThreads;
  const int64_t b = threadIdx.x * per;
  const int64_t e = b + per < ntiles ? b + per : ntiles;
  S acc{};
  for (int64_t t = b; t < e; ++t) acc = combine(op, acc, load_state(ts, o + t, ts.f[t]));
  S total;
  S run = block_exclusive<T::kCarryThreads / 32, false, S>(op, acc, warp_tot, &total);
  for (int64_t t = b; t < e; ++t) {
    const S x = load_state(ts, o + t, ts.f[t]);
    store_state(ts, o + t, run);
    run = combine(op, run, x);
  }
}

int64_t num_tiles(int64_t nrows) { return (nrows + kTile - 1) / kTile; }

template <class T>
size_t segscan_scratch_bytes(int64_t nrows, int ncols) {
  if (nrows <= 0 || ncols <= 0) return 0;
  return (size_t)num_tiles(nrows) * (8 * T::State::kWords * (size_t)ncols + 4);
}

template <class T, bool kReverse = false, bool kBlocks = false>
int launch_segscan(cudaStream_t st, int64_t block, int64_t nrows, int64_t nseg, const int64_t* offsets,
                   const typename T::Cols& a, void* scratch) {
  const int64_t ntiles = num_tiles(nrows);
  const TileStates<typename T::State> ts = tile_states<typename T::State>(scratch, a.ncols * ntiles);
  const unsigned grid = (unsigned)ntiles;
  fb_segscan_tile_kernel<T, false, kReverse, kBlocks><<<grid, kThreads, 0, st>>>(nrows, nseg, offsets, a, ntiles,
                                                                                  ts, block);
  FB_CUDA(cudaGetLastError());
  fb_segscan_carry_kernel<T><<<a.ncols, T::kCarryThreads, 0, st>>>(ntiles, a, ts);
  FB_CUDA(cudaGetLastError());
  fb_segscan_tile_kernel<T, true, kReverse, kBlocks><<<grid, kThreads, 0, st>>>(nrows, nseg, offsets, a, ntiles,
                                                                                 ts, block);
  FB_CUDA(cudaGetLastError());
  return 0;
}

// one inclusive scan of every column into its outputs; with T::kFrames, reversed (S) and / or restarting at blocks
// of `block` rows (block > 0)
template <class T>
int run_segscan(cudaStream_t st, bool reverse, int64_t block, int64_t nrows, int64_t nseg, const int64_t* offsets,
                const typename T::Cols& a, void* scratch) {
  if constexpr (T::kFrames) {
    if (reverse && block > 0) return launch_segscan<T, true, true>(st, block, nrows, nseg, offsets, a, scratch);
    if (reverse) return launch_segscan<T, true>(st, block, nrows, nseg, offsets, a, scratch);
    if (block > 0) return launch_segscan<T, false, true>(st, block, nrows, nseg, offsets, a, scratch);
  }
  return launch_segscan<T>(st, block, nrows, nseg, offsets, a, scratch);
}

// ---- moving frames -------------------------------------------------------------------------------
constexpr int kFrameThreads = 256;
constexpr int kFrameItems = 8;                          // consecutive staged rows per thread
constexpr int kFrameSpan = kFrameThreads * kFrameItems;  // staged rows per CTA: outputs + W - 1 halo
static_assert(2 * FB_FRAME_TILE_MAX_WIDTH == kFrameSpan, "a CTA at the widest frame writes about half its span");
static_assert(kFrameItems == 8, "padded() assumes 8 rows per thread");

// which of P[hi] / S[lo] make up a row's frame; packed with lo and hi (staged indices, 11 bits each)
enum : uint32_t { kFrameEmpty = 0, kFrameP = 1, kFrameS = 2, kFrameBoth = 3 };

__device__ __forceinline__ uint32_t frame_code(int lo, int hi, int blk_lo, int blk_hi, int p_start) {
  const uint32_t mode = blk_lo != blk_hi ? kFrameBoth : (lo == p_start ? kFrameP : kFrameS);
  return mode | (uint32_t)lo << 2 | (uint32_t)hi << 13;
}

// Row i's ROWS frame [lo, hi] inside its segment [sa, sb) (lo > hi: empty), with start / end clipped by make_frame
// so that i + start and i + end cannot wrap.  The combine pass and fb_window_value both call it.
__device__ __forceinline__ void rows_frame(int64_t i, int64_t sa, int64_t sb, int64_t start, int64_t end, int flags,
                                           int64_t* lo, int64_t* hi) {
  *lo = (flags & FB_FRAME_UNBOUNDED_START) || i + start < sa ? sa : i + start;
  *hi = (flags & FB_FRAME_UNBOUNDED_END) || i + end > sb - 1 ? sb - 1 : i + end;
}

struct FrameSmem {
  uint64_t pv[padded(kFrameSpan)];  // staged values, then P
  uint64_t sv[padded(kFrameSpan)];
  int32_t pc[padded(kFrameSpan)];   // a frame has at most kFrameSpan rows: int32 counts
  int32_t sc[padded(kFrameSpan)];
  uint8_t valid[kFrameSpan];
  uint8_t heads[kFrameSpan];        // bit 0: a P run starts at the row; bit 1: an S run ends at it
  uint8_t seg_head[kFrameSpan + 1];
  St warp_tot[kFrameThreads / 32];
  int64_t range[4];
};

// One CTA per `per_tile` output rows [o0, o1): stage rows [s0, s1) = [o0 + start, o1 + end) clipped to the
// table (every frame of the tile lies inside), scan P and S there, write value and count once.
__global__ void __launch_bounds__(kFrameThreads)
fb_window_frame_tile_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                            const __grid_constant__ ScanCols a, int64_t start, int width, int64_t per_tile) {
  extern __shared__ __align__(16) unsigned char frame_smem[];
  FrameSmem& sm = *reinterpret_cast<FrameSmem*>(frame_smem);
  const int64_t end = start + width - 1;
  const int64_t o0 = (int64_t)blockIdx.x * per_tile;
  const int64_t o1 = o0 + per_tile < nrows ? o0 + per_tile : nrows;
  const int64_t s0 = o0 + start > 0 ? o0 + start : 0;
  const int64_t s1 = o1 + end < nrows ? o1 + end : nrows;
  const int nloc = s1 > s0 ? (int)(s1 - s0) : 0;
  // ---- segments: starts inside [s0, s1] marked in shared memory; the segments of the output rows
  for (int i = threadIdx.x; i <= kFrameSpan; i += kFrameThreads) sm.seg_head[i] = 0;
  if (threadIdx.x == 0) {
    sm.range[0] = lower_bound(offsets, nseg + 1, s0);
    sm.range[1] = upper_bound(offsets, nseg + 1, s1);
    sm.range[2] = upper_bound(offsets, nseg + 1, o0) - 1;      // segment of o0
    sm.range[3] = upper_bound(offsets, nseg + 1, o1 - 1) + 1;  // one past the offset ending o1 - 1's segment
  }
  __syncthreads();
  for (int64_t s = sm.range[0] + threadIdx.x; s < sm.range[1]; s += kFrameThreads)
    sm.seg_head[__ldg(offsets + s) - s0] = 1;
  __syncthreads();
  const int64_t m0 = first_multiple(s0, width);
  const int rem0 = m0 == s0 ? 0 : (int)(s0 - (m0 - width));  // s0 % W: blocks are aligned to multiples of W
  for (int j = threadIdx.x; j < kFrameSpan; j += kFrameThreads) {
    const bool p = sm.seg_head[j] || (rem0 + j) % width == 0;
    const bool s = j + 1 >= nloc || sm.seg_head[j + 1] || (rem0 + j + 1) % width == 0;
    sm.heads[j] = (uint8_t)(p | s << 1);
  }
  // ---- every output row's frame [lo, hi] in staged rows; thread t has rows o0 + t + kFrameThreads * k
  uint32_t code[kFrameItems];
  const int64_t q0 = sm.range[2], nq = sm.range[3] - q0;
#pragma unroll
  for (int k = 0; k < kFrameItems; ++k) {
    const int64_t i = o0 + threadIdx.x + (int64_t)kFrameThreads * k;
    code[k] = kFrameEmpty;
    if (i >= o1) continue;
    const int64_t q = q0 + upper_bound(offsets + q0, nq, i) - 1;
    const int64_t sa = __ldg(offsets + q), sb = __ldg(offsets + q + 1);
    const int64_t lo = i + start > sa ? i + start : sa;
    const int64_t hi = i + end < sb - 1 ? i + end : sb - 1;
    if (lo > hi) continue;
    const int jl = (int)(lo - s0), jh = (int)(hi - s0);  // staged rows
    const int bs = jh - (rem0 + jh) % width;                // start of hi's block
    const int ja = sa > s0 ? (int)(sa - s0) : 0;            // segment start, or the first staged row
    const int ps = bs > ja ? bs : ja;                       // where P[hi]'s run starts
    code[k] = frame_code(jl, jh, (rem0 + jl) / width, (rem0 + jh) / width, ps);
  }
  const int j0 = threadIdx.x * kFrameItems;
  for (int col = 0; col < a.ncols; ++col) {
    const int op = a.op[col];
    const bool is_count = op == FB_AGG_COUNT;
    const uint64_t* __restrict__ src = (const uint64_t*)a.vals[col];
    const uint8_t* __restrict__ vm = a.valid[col];
    for (int i = threadIdx.x; i < kFrameSpan; i += kFrameThreads) {
      const bool in = i < nloc;
      if (!is_count) sm.pv[padded(i)] = in ? __ldg((const unsigned long long*)src + s0 + i) : 0;
      sm.valid[i] = in ? (vm == nullptr ? 1 : (__ldg(vm + s0 + i) != 0)) : 0;
    }
    __syncthreads();
    uint64_t x[kFrameItems];
    uint32_t ok = 0, hd = 0;
#pragma unroll
    for (int k = 0; k < kFrameItems; ++k) {
      const int j = j0 + k;
      x[k] = is_count ? 0 : sm.pv[padded(j)];
      ok |= (uint32_t)(sm.valid[j] != 0) << k;
      hd |= (uint32_t)sm.heads[j] << (2 * k);
    }
    // P: forward over the staged rows
    St acc{0, 0, 0}, total;
#pragma unroll
    for (int k = 0; k < kFrameItems; ++k) {
      const int c = (ok >> k) & 1;
      acc = combine(op, acc, St{c ? x[k] : 0, c, (int32_t)((hd >> (2 * k)) & 1)});
    }
    St run = block_exclusive<kFrameThreads / 32>(op, acc, sm.warp_tot, &total);  // all x[] read before pv is written
#pragma unroll
    for (int k = 0; k < kFrameItems; ++k) {
      const int c = (ok >> k) & 1;
      run = combine(op, run, St{c ? x[k] : 0, c, (int32_t)((hd >> (2 * k)) & 1)});
      sm.pv[padded(j0 + k)] = run.c > 0 ? run.v : 0;
      sm.pc[padded(j0 + k)] = (int32_t)run.c;
    }
    // S: backward
    acc = St{0, 0, 0};
#pragma unroll
    for (int k = kFrameItems - 1; k >= 0; --k) {
      const int c = (ok >> k) & 1;
      acc = combine(op, acc, St{c ? x[k] : 0, c, (int32_t)((hd >> (2 * k + 1)) & 1)});
    }
    run = block_exclusive<kFrameThreads / 32, true>(op, acc, sm.warp_tot, &total);
#pragma unroll
    for (int k = kFrameItems - 1; k >= 0; --k) {
      const int c = (ok >> k) & 1;
      run = combine(op, run, St{c ? x[k] : 0, c, (int32_t)((hd >> (2 * k + 1)) & 1)});
      sm.sv[padded(j0 + k)] = run.c > 0 ? run.v : 0;
      sm.sc[padded(j0 + k)] = (int32_t)run.c;
    }
    __syncthreads();
    uint64_t* __restrict__ ov = (uint64_t*)a.out_vals[col];
    int64_t* __restrict__ oc = a.out_count[col];
#pragma unroll
    for (int k = 0; k < kFrameItems; ++k) {
      const int64_t i = o0 + threadIdx.x + (int64_t)kFrameThreads * k;
      if (i >= o1) break;
      const uint32_t mode = code[k] & 3;
      const int lo = (int)((code[k] >> 2) & 0x7FF), hi = (int)((code[k] >> 13) & 0x7FF);
      St r{0, 0, 0};
      if (mode & kFrameS) r = St{sm.sv[padded(lo)], sm.sc[padded(lo)], 0};
      if (mode & kFrameP) r = combine(op, r, St{sm.pv[padded(hi)], sm.pc[padded(hi)], 0});
      if (ov != nullptr) ov[i] = r.c > 0 ? r.v : 0;
      if (oc != nullptr) oc[i] = r.c;
    }
    __syncthreads();  // shared buffers are refilled by the next column
  }
}

// The frames from P and S in scratch (pv / pc / sv / sc: ncols x nrows; P or S unused with an unbounded
// side).  width == 0: no blocks.  One CTA per kTile rows.
__global__ void __launch_bounds__(kThreads)
fb_window_frame_combine_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                               const __grid_constant__ ScanCols a, int64_t start, int64_t end, int flags,
                               int64_t width, const uint64_t* __restrict__ pv, const int64_t* __restrict__ pc,
                               const uint64_t* __restrict__ sv, const int64_t* __restrict__ sc) {
  __shared__ int64_t range[2];
  const int64_t t0 = (int64_t)blockIdx.x * kTile;
  const int64_t t1 = t0 + kTile < nrows ? t0 + kTile : nrows;
  if (threadIdx.x == 0) {
    range[0] = upper_bound(offsets, nseg + 1, t0) - 1;
    range[1] = upper_bound(offsets, nseg + 1, t1 - 1) + 1;
  }
  __syncthreads();
  const int64_t q0 = range[0], nq = range[1] - q0;
  for (int64_t i = t0 + threadIdx.x; i < t1; i += kThreads) {
    const int64_t q = q0 + upper_bound(offsets + q0, nq, i) - 1;
    const int64_t sa = __ldg(offsets + q), sb = __ldg(offsets + q + 1);
    int64_t lo, hi;
    rows_frame(i, sa, sb, start, end, flags, &lo, &hi);
    uint32_t mode = kFrameEmpty;
    if (lo <= hi) {
      if (flags & FB_FRAME_UNBOUNDED_START) mode = kFrameP;
      else if (flags & FB_FRAME_UNBOUNDED_END) mode = kFrameS;
      else {
        const int64_t bs = hi - hi % width;
        mode = lo / width != hi / width ? kFrameBoth : (lo == (bs > sa ? bs : sa) ? kFrameP : kFrameS);
      }
    }
    for (int col = 0; col < a.ncols; ++col) {
      const int op = a.op[col];
      const int64_t base = col * nrows;
      St r{0, 0, 0};
      if (mode & kFrameS) r = St{sv[base + lo], sc[base + lo], 0};
      if (mode & kFrameP) r = combine(op, r, St{pv[base + hi], pc[base + hi], 0});
      if (a.out_vals[col] != nullptr) ((uint64_t*)a.out_vals[col])[i] = r.c > 0 ? r.v : 0;
      if (a.out_count[col] != nullptr) a.out_count[col][i] = r.c;
    }
  }
}

// A frame on `nrows` rows, bounds clipped to [-nrows, nrows] (no sum below overflows) and a bound that
// reaches past every segment made unbounded: both exact, as no segment is longer than the table.
struct Frame {
  int64_t start, end, width;  // width: end - start + 1 with both sides bounded, else 0
  int flags;
  bool tile;                  // the one-pass path
};

Frame make_frame(int64_t nrows, int64_t start, int64_t end, int flags) {
  Frame f;
  f.flags = flags & (FB_FRAME_UNBOUNDED_START | FB_FRAME_UNBOUNDED_END);
  f.start = start < -nrows ? -nrows : (start > nrows ? nrows : start);
  f.end = end < -nrows ? -nrows : (end > nrows ? nrows : end);
  if (f.start <= -nrows) f.flags |= FB_FRAME_UNBOUNDED_START;
  if (f.end >= nrows) f.flags |= FB_FRAME_UNBOUNDED_END;
  f.width = f.flags == 0 ? f.end - f.start + 1 : 0;
  f.tile = f.flags == 0 && f.width <= FB_FRAME_TILE_MAX_WIDTH;
  return f;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t frame_scratch(int64_t nrows, int ncols, const Frame& f) {
  if (nrows <= 0 || ncols <= 0 || f.tile) return 0;
  const int sides = f.flags == 0 ? 2 : 1;
  return align256(segscan_scratch_bytes<OpScan>(nrows, ncols)) + (size_t)sides * 16 * ncols * (size_t)nrows;
}

// ---- value frames (RANGE BETWEEN) ----------------------------------------------------------------
constexpr int kRangeThreads = 256;  // one row per thread: neighbouring rows search neighbouring keys

// The presort key as an unsigned order key, as sort._unsigned_order_key builds it: sign bit flipped for
// signed integers, the value itself for unsigned ones, the total-order transform for f64 (-0.0 read as 0.0).
__device__ __forceinline__ uint64_t range_order_bits(uint64_t k, int cls) {
  if (cls == FB_RANGE_KEY_I64) return k ^ 0x8000000000000000ULL;
  if (cls == FB_RANGE_KEY_U64) return k;
  if (__longlong_as_double((long long)k) == 0.0) k = 0;
  return (int64_t)k < 0 ? ~k : k ^ 0x8000000000000000ULL;
}

// A bound key k + off (ASC) or k - off (DESC) in the searched order (ASC: the order key, DESC: its
// complement, so that the non-NULL run of a segment is ascending either way).  inf = -1 / +1: below /
// above every key of the type (an integer sum past the type's range); then v is unused.
struct RangeTarget {
  uint64_t v;
  int inf;
};

__device__ __forceinline__ RangeTarget range_target(uint64_t k, uint64_t off, int cls, bool desc) {
  RangeTarget t{0, 0};
  if (cls == FB_RANGE_KEY_F64) {  // one IEEE addition, round to nearest even; overflow gives +-inf, a key
    const double o = __longlong_as_double((long long)off);
    const double x = __longlong_as_double((long long)k) + (desc ? -o : o);
    t.v = range_order_bits((uint64_t)__double_as_longlong(x), cls);
  } else {  // exact: 128-bit sum, compared with the type's range
    const __int128 kk = cls == FB_RANGE_KEY_I64 ? (__int128)(int64_t)k : (__int128)k;
    const __int128 oo = (__int128)(int64_t)off;
    const __int128 x = desc ? kk - oo : kk + oo;
    const __int128 lo = cls == FB_RANGE_KEY_I64 ? -((__int128)1 << 63) : (__int128)0;
    const __int128 hi = cls == FB_RANGE_KEY_I64 ? ((__int128)1 << 63) - 1 : ((__int128)1 << 64) - 1;
    if (x < lo) t.inf = -1;
    else if (x > hi) t.inf = 1;
    else t.v = range_order_bits((uint64_t)x, cls);
  }
  if (desc) {
    t.v = ~t.v;
    t.inf = -t.inf;
  }
  return t;
}

// First row j of [a, e) with key(j) >= t (kStrict: key(j) > t) in the searched order, e if none.  The
// non-NULL run [a, e) is sorted, so this is a lower_bound (upper_bound when kStrict) over it, found by
// galloping from row i in [a, e): O(log |answer - i|) loads, not O(log (e - a)).
template <bool kStrict>
__device__ __forceinline__ int64_t range_search(const uint64_t* __restrict__ keys, int cls, bool desc, int64_t a,
                                                int64_t e, int64_t i, const RangeTarget& t) {
  if (t.inf < 0) return a;
  if (t.inf > 0) return e;
  auto hit = [&](int64_t j) {
    uint64_t o = range_order_bits(__ldg((const unsigned long long*)keys + j), cls);
    if (desc) o = ~o;
    return kStrict ? o > t.v : o >= t.v;
  };
  int64_t lo, hi;  // hit() is false on [a, lo) and true on [hi, e): the answer is in [lo, hi]
  if (hit(i)) {
    hi = i;
    lo = a;
    for (int64_t step = 1;; step <<= 1) {
      const int64_t j = hi - step;
      if (j < a) break;
      if (!hit(j)) { lo = j + 1; break; }
      hi = j;
    }
  } else {
    lo = i + 1;
    hi = e;
    for (int64_t step = 1;; step <<= 1) {
      const int64_t j = lo - 1 + step;
      if (j >= e) break;
      if (hit(j)) { hi = j; break; }
      lo = j + 1;
    }
  }
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (hit(m)) hi = m; else lo = m + 1;
  }
  return lo;
}

// first NULL-key row of every segment (its NULL rows are its tail): a binary search on the validity bytes
__global__ void __launch_bounds__(kRangeThreads)
fb_range_null_start_kernel(int64_t nseg, const int64_t* __restrict__ offsets, const uint8_t* __restrict__ valid,
                           int64_t* __restrict__ null_start) {
  const int64_t s = (int64_t)blockIdx.x * kRangeThreads + threadIdx.x;
  if (s >= nseg) return;
  int64_t lo = __ldg(offsets + s), hi = __ldg(offsets + s + 1);
  if (valid == nullptr) lo = hi;  // no NULL keys
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (__ldg(valid + m) != 0) lo = m + 1; else hi = m;
  }
  null_start[s] = lo;
}

__global__ void __launch_bounds__(kRangeThreads)
fb_range_bounds_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                       const int64_t* __restrict__ null_start, const uint64_t* __restrict__ keys, int cls, int desc,
                       uint64_t start, uint64_t end, int flags, int64_t* __restrict__ out_lo,
                       int64_t* __restrict__ out_hi) {
  __shared__ int64_t range[2];
  const int64_t t0 = (int64_t)blockIdx.x * kRangeThreads;
  const int64_t t1 = t0 + kRangeThreads < nrows ? t0 + kRangeThreads : nrows;
  if (threadIdx.x == 0) {
    range[0] = upper_bound(offsets, nseg + 1, t0) - 1;
    range[1] = upper_bound(offsets, nseg + 1, t1 - 1) + 1;
  }
  __syncthreads();
  const int64_t i = t0 + threadIdx.x;
  if (i >= t1) return;
  const int64_t q0 = range[0];
  const int64_t q = q0 + upper_bound(offsets + q0, range[1] - q0, i) - 1;
  const int64_t a = __ldg(offsets + q), b = __ldg(offsets + q + 1), e = __ldg(null_start + q);
  int64_t lo, hi;
  if (i >= e) {  // a NULL key: its peers are the NULL tail [e, b)
    lo = (flags & FB_FRAME_UNBOUNDED_START) ? a : e;
    hi = b - 1;
  } else {
    const uint64_t k = __ldg((const unsigned long long*)keys + i);
    if (flags & FB_FRAME_UNBOUNDED_START) lo = a;
    else lo = range_search<false>(keys, cls, desc != 0, a, e, i, range_target(k, start, cls, desc != 0));
    if (flags & FB_FRAME_UNBOUNDED_END) hi = b - 1;
    else hi = range_search<true>(keys, cls, desc != 0, a, e, i, range_target(k, end, cls, desc != 0)) - 1;
  }
  out_lo[i] = lo;
  out_hi[i] = hi;
}

// ---- aggregates over arbitrary row intervals: an aligned power-of-two block tree ----------------------
// Level l >= 1 holds (op, count) of rows [m 2^l, (m + 1) 2^l) for m < nrows >> l, in scratch; level 0 is the
// input.  Level l starts at node tree_off[l] of a column's nodes (TreeLevels, fb_tree.cuh).

__device__ __forceinline__ St tree_node(const ScanCols& a, int col, bool is_count, const TreeLevels& L,
                                        const uint64_t* __restrict__ tv, const int64_t* __restrict__ tc, int level,
                                        int64_t m) {
  if (level == 0) {
    const uint8_t* vm = a.valid[col];
    const int c = vm == nullptr ? 1 : (__ldg(vm + m) != 0);
    return St{c && !is_count ? __ldg((const unsigned long long*)a.vals[col] + m) : 0, c, 0};
  }
  const int64_t p = (int64_t)col * L.total + L.off[level] + m;
  return St{is_count ? 0 : __ldg((const unsigned long long*)tv + p), __ldg((const long long*)tc + p), 0};
}

// one level of the tree from the one below, pairwise in a fixed order; blockIdx.y = column
__global__ void __launch_bounds__(kThreads)
fb_tree_level_kernel(const __grid_constant__ ScanCols a, const __grid_constant__ TreeLevels L, int level,
                     int64_t nrows, uint64_t* __restrict__ tv, int64_t* __restrict__ tc) {
  const int col = blockIdx.y;
  const int op = a.op[col];
  const bool is_count = op == FB_AGG_COUNT;
  const int64_t nodes = nrows >> level;
  for (int64_t m = (int64_t)blockIdx.x * kThreads + threadIdx.x; m < nodes; m += (int64_t)gridDim.x * kThreads) {
    const St r = combine(op, tree_node(a, col, is_count, L, tv, tc, level - 1, 2 * m),
                         tree_node(a, col, is_count, L, tv, tc, level - 1, 2 * m + 1));
    const int64_t p = (int64_t)col * L.total + L.off[level] + m;
    if (!is_count) tv[p] = r.c > 0 ? r.v : 0;
    tc[p] = r.c;
  }
}

// Per row, [lo, hi] clamped to [0, nrows) as its canonical decomposition into tree blocks (at most two per
// level, O(log width) levels), combined left to right.
__global__ void __launch_bounds__(kThreads)
fb_tree_query_kernel(const __grid_constant__ ScanCols a, const __grid_constant__ TreeLevels L, int64_t nrows,
                     const int64_t* __restrict__ d_lo, const int64_t* __restrict__ d_hi,
                     const uint64_t* __restrict__ tv, const int64_t* __restrict__ tc) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= nrows) return;
  int64_t lo = __ldg((const long long*)d_lo + i), hi = __ldg((const long long*)d_hi + i);
  lo = lo < 0 ? 0 : lo;
  hi = hi > nrows - 1 ? nrows - 1 : hi;
  for (int col = 0; col < a.ncols; ++col) {
    const int op = a.op[col];
    const bool is_count = op == FB_AGG_COUNT;
    St left{0, 0, 0}, right{0, 0, 0};
    int64_t l = lo, r = hi + 1;  // [l, r) in blocks of the current level
    for (int level = 0; l < r; ++level, l >>= 1, r >>= 1) {
      if (l & 1) left = combine(op, left, tree_node(a, col, is_count, L, tv, tc, level, l++));
      if (r & 1) right = combine(op, tree_node(a, col, is_count, L, tv, tc, level, --r), right);
    }
    const St res = combine(op, left, right);
    if (a.out_vals[col] != nullptr) ((uint64_t*)a.out_vals[col])[i] = res.c > 0 ? res.v : 0;
    if (a.out_count[col] != nullptr) a.out_count[col][i] = res.c;
  }
}

// levels 1.. of the tree of every column of `a` into scratch (values, then counts), one launch per level
int build_tree(int dev, cudaStream_t st, const ScanCols& a, int64_t nrows, void* scratch) {
  const TreeLevels L = tree_levels(nrows);
  uint64_t* tv = (uint64_t*)scratch;
  int64_t* tc = (int64_t*)(tv + (size_t)a.ncols * L.total);
  const int64_t max_grid = 8 * (int64_t)fb_sm_count(dev);
  for (int level = 1; level <= L.levels; ++level) {
    const int64_t blocks = ((nrows >> level) + kThreads - 1) / kThreads;
    const dim3 grid((unsigned)(blocks < max_grid ? blocks : max_grid), (unsigned)a.ncols);
    fb_tree_level_kernel<<<grid, kThreads, 0, st>>>(a, L, level, nrows, tv, tc);
    FB_CUDA(cudaGetLastError());
  }
  return 0;
}

// ---- value heads: FIRST_VALUE / LAST_VALUE / NTH_VALUE ------------------------------------------------
struct ValueCols {
  const void* vals[FB_SCAN_MAX_COLS];
  const uint8_t* valid[FB_SCAN_MAX_COLS];
  void* out[FB_SCAN_MAX_COLS];
  uint8_t* out_valid[FB_SCAN_MAX_COLS];
  int64_t nth[FB_SCAN_MAX_COLS];  // >= 1: the frame's nth row (at most nrows + 1); FB_VALUE_LAST: its last row
  int32_t width[FB_SCAN_MAX_COLS];
  int32_t ncols;
};

// One thread per row: the row's frame (ROWS: rows_frame over its segment; else [d_lo, d_hi] clamped to the table),
// the picked row, then every column's value and validity at that row.  Neighbouring rows pick neighbouring rows.
__global__ void __launch_bounds__(kRangeThreads)
fb_window_value_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets, int64_t start, int64_t end,
                       int flags, const int64_t* __restrict__ d_lo, const int64_t* __restrict__ d_hi,
                       const __grid_constant__ ValueCols a) {
  __shared__ int64_t range[2];
  const int64_t t0 = (int64_t)blockIdx.x * kRangeThreads;
  const int64_t t1 = t0 + kRangeThreads < nrows ? t0 + kRangeThreads : nrows;
  const int64_t i = t0 + threadIdx.x;
  int64_t lo, hi;
  if (d_lo == nullptr) {  // uniform across the CTA
    if (threadIdx.x == 0) {
      range[0] = upper_bound(offsets, nseg + 1, t0) - 1;
      range[1] = upper_bound(offsets, nseg + 1, t1 - 1) + 1;
    }
    __syncthreads();
    if (i >= t1) return;
    const int64_t q0 = range[0];
    const int64_t q = q0 + upper_bound(offsets + q0, range[1] - q0, i) - 1;
    rows_frame(i, __ldg(offsets + q), __ldg(offsets + q + 1), start, end, flags, &lo, &hi);
  } else {
    if (i >= t1) return;
    lo = __ldg((const long long*)d_lo + i);
    hi = __ldg((const long long*)d_hi + i);
    lo = lo < 0 ? 0 : lo;
    hi = hi > nrows - 1 ? nrows - 1 : hi;
  }
  for (int c = 0; c < a.ncols; ++c) {
    const int64_t n = a.nth[c];
    const int64_t j = n == FB_VALUE_LAST ? hi : lo + n - 1;  // lo <= nrows and n <= nrows + 1: no wrap
    const bool hit = lo <= hi && j <= hi;
    const uint8_t* vm = a.valid[c];
    const bool ok = hit && (vm == nullptr || __ldg(vm + j) != 0);
    switch (a.width[c]) {
      case 1: ((uint8_t*)a.out[c])[i] = ok ? __ldg((const uint8_t*)a.vals[c] + j) : 0; break;
      case 2: ((uint16_t*)a.out[c])[i] = ok ? __ldg((const unsigned short*)a.vals[c] + j) : 0; break;
      case 4: ((uint32_t*)a.out[c])[i] = ok ? __ldg((const unsigned int*)a.vals[c] + j) : 0; break;
      default: ((uint64_t*)a.out[c])[i] = ok ? __ldg((const unsigned long long*)a.vals[c] + j) : 0; break;
    }
    a.out_valid[c][i] = ok ? 1 : 0;
  }
}

// ---- distribution heads: PERCENT_RANK / CUME_DIST / NTILE ---------------------------------------------
// A peer group is the rows from one head byte to the next (or to its segment's bound).  Head bytes are not
// monotone, so no search over them bounds its loads by the distance; instead each tile of kTile rows publishes
// the first and last head row inside it, one CTA turns those into the last head before every tile and the first
// head after it (a max / min scan over tiles), and the row pass resolves every row's peer group from its tile's
// heads in shared memory plus those two carries: O(1) per row whatever the size of the peer group.
struct DistCols {
  int64_t n[FB_SCAN_MAX_COLS];
  int64_t* out[FB_SCAN_MAX_COLS];
  int32_t ncols;
};

constexpr int64_t kNoHead = INT64_MAX;

__device__ __forceinline__ int64_t max64(int64_t a, int64_t b) { return a > b ? a : b; }
__device__ __forceinline__ int64_t min64(int64_t a, int64_t b) { return a < b ? a : b; }

// Per tile: the first head row in it (kNoHead: none) and the last (-1: none).
__global__ void __launch_bounds__(kThreads)
fb_peer_tile_kernel(int64_t nrows, const uint8_t* __restrict__ heads, int64_t* __restrict__ tile_first,
                    int64_t* __restrict__ tile_last) {
  __shared__ int64_t wf[kThreads / 32], wl[kThreads / 32];
  const int64_t t0 = (int64_t)blockIdx.x * kTile;
  int64_t f = kNoHead, l = -1;
  for (int k = 0; k < kItems; ++k) {
    const int64_t i = t0 + threadIdx.x + (int64_t)kThreads * k;
    if (i < nrows && __ldg(heads + i) != 0) {
      f = min64(f, i);
      l = i;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    f = min64(f, __shfl_xor_sync(0xFFFFFFFFu, f, d));
    l = max64(l, __shfl_xor_sync(0xFFFFFFFFu, l, d));
  }
  if ((threadIdx.x & 31) == 0) {
    wf[threadIdx.x >> 5] = f;
    wl[threadIdx.x >> 5] = l;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) {
      f = min64(f, wf[w]);
      l = max64(l, wl[w]);
    }
    tile_first[blockIdx.x] = min64(f, wf[0]);
    tile_last[blockIdx.x] = max64(l, wl[0]);
  }
}

constexpr int kCarryThreads = 1024;

// One CTA, in place: tile_last[t] := the last head row before tile t (-1: none), tile_first[t] := the first head row
// after it (kNoHead: none).  Thread k owns a contiguous run of tiles; the runs' totals are scanned in shared memory.
__global__ void __launch_bounds__(kCarryThreads, 1)
fb_peer_carry_kernel(int64_t ntiles, int64_t* __restrict__ tile_first, int64_t* __restrict__ tile_last) {
  __shared__ int64_t sl[kCarryThreads], sf[kCarryThreads];
  const int64_t per = (ntiles + kCarryThreads - 1) / kCarryThreads;
  const int64_t b0 = min64((int64_t)threadIdx.x * per, ntiles), b1 = min64(b0 + per, ntiles);
  int64_t l = -1, f = kNoHead;
  for (int64_t t = b0; t < b1; ++t) {
    l = max64(l, tile_last[t]);
    f = min64(f, tile_first[t]);
  }
  sl[threadIdx.x] = l;
  sf[threadIdx.x] = f;
  __syncthreads();
  for (int d = 1; d < kCarryThreads; d <<= 1) {  // inclusive: max from the left, min from the right
    const int k = threadIdx.x;
    const int64_t xl = k >= d ? sl[k - d] : -1;
    const int64_t xf = k + d < kCarryThreads ? sf[k + d] : kNoHead;
    __syncthreads();
    sl[k] = max64(sl[k], xl);
    sf[k] = min64(sf[k], xf);
    __syncthreads();
  }
  l = threadIdx.x > 0 ? sl[threadIdx.x - 1] : -1;
  f = threadIdx.x + 1 < kCarryThreads ? sf[threadIdx.x + 1] : kNoHead;
  for (int64_t t = b0; t < b1; ++t) {
    const int64_t x = tile_last[t];
    tile_last[t] = l;
    l = max64(l, x);
  }
  for (int64_t t = b1 - 1; t >= b0; --t) {
    const int64_t x = tile_first[t];
    tile_first[t] = f;
    f = min64(f, x);
  }
}

// Max (kRev: min) over the threads before (kRev: after) this one of x, and of seed: exact and order-free.
template <bool kRev>
__device__ __forceinline__ int64_t block_exclusive_extreme(int64_t x, int64_t seed, int64_t* warp_tot) {
  constexpr int kWarps = kThreads / 32;
  const int lane = kRev ? 31 - (threadIdx.x & 31) : threadIdx.x & 31;
  const int w = kRev ? kWarps - 1 - (int)(threadIdx.x >> 5) : threadIdx.x >> 5;
  auto op = [](int64_t p, int64_t q) { return kRev ? min64(p, q) : max64(p, q); };
  int64_t inc = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int64_t o = kRev ? __shfl_down_sync(0xFFFFFFFFu, inc, d) : __shfl_up_sync(0xFFFFFFFFu, inc, d);
    if (lane >= d) inc = op(inc, o);
  }
  const int64_t ex = kRev ? __shfl_down_sync(0xFFFFFFFFu, inc, 1) : __shfl_up_sync(0xFFFFFFFFu, inc, 1);
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  int64_t pre = seed;
  for (int k = 0; k < w; ++k) pre = op(pre, warp_tot[k]);
  __syncthreads();  // warp_tot is reused by the next call
  return lane == 0 ? pre : op(pre, ex);
}

// One CTA per kTile rows.  Thread t reads head bytes of rows 8t .. 8t + 7 of the tile from shared memory and finds
// every row's last head at or before it and first head after it; then rows are striped over threads for the
// segment search and the coalesced stores.
__global__ void __launch_bounds__(kThreads)
fb_window_distribution_kernel(int64_t nrows, int64_t nseg, const int64_t* __restrict__ offsets,
                              const uint8_t* __restrict__ heads, const int64_t* __restrict__ tile_first,
                              const int64_t* __restrict__ tile_last, double* __restrict__ percent_rank,
                              double* __restrict__ cume_dist, const __grid_constant__ DistCols d) {
  __shared__ uint8_t hd[kTile];
  __shared__ int64_t pf[kTile], nx[kTile];
  __shared__ int64_t warp_tot[kThreads / 32];
  __shared__ int64_t range[2];
  const int64_t t0 = (int64_t)blockIdx.x * kTile;
  const int64_t t1 = t0 + kTile < nrows ? t0 + kTile : nrows;
  if (threadIdx.x == 0) {
    range[0] = upper_bound(offsets, nseg + 1, t0) - 1;
    range[1] = upper_bound(offsets, nseg + 1, t1 - 1) + 1;
  }
  for (int j = threadIdx.x; j < kTile; j += kThreads) hd[j] = t0 + j < t1 ? __ldg(heads + t0 + j) : 0;
  __syncthreads();
  const int j0 = threadIdx.x * kItems;
  int64_t last = -1, first = kNoHead;
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    if (hd[j0 + k]) {
      last = t0 + j0 + k;
      first = min64(first, t0 + j0 + k);
    }
  }
  int64_t p = block_exclusive_extreme<false>(last, tile_last[blockIdx.x], warp_tot);
  int64_t q = block_exclusive_extreme<true>(first, tile_first[blockIdx.x], warp_tot);
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    if (hd[j0 + k]) p = t0 + j0 + k;
    pf[j0 + k] = p;
  }
#pragma unroll
  for (int k = kItems - 1; k >= 0; --k) {
    nx[j0 + k] = q;
    if (hd[j0 + k]) q = t0 + j0 + k;
  }
  __syncthreads();
  const int64_t q0 = range[0], nq = range[1] - q0;
  for (int j = threadIdx.x; j < kTile; j += kThreads) {
    const int64_t i = t0 + j;
    if (i >= t1) break;
    const int64_t s = q0 + upper_bound(offsets + q0, nq, i) - 1;
    const int64_t a = __ldg(offsets + s), b = __ldg(offsets + s + 1);
    const int64_t first_peer = max64(pf[j], a), last_peer = min64(nx[j], b) - 1;
    const int64_t rows = b - a;
    if (percent_rank != nullptr)  // (rank - 1) / (N - 1): one IEEE division of two exact integers
      percent_rank[i] = rows > 1 ? (double)(first_peer - a) / (double)(rows - 1) : 0.0;
    if (cume_dist != nullptr) cume_dist[i] = (double)(last_peer - a + 1) / (double)rows;
    const int64_t r = i - a;
    for (int c = 0; c < d.ncols; ++c) {  // SQLite's NTILE: N / n rows a bucket, the first N % n buckets one more
      const int64_t n = d.n[c], size = rows / n;
      int64_t bucket;
      if (size == 0) {
        bucket = r + 1;
      } else {
        const int64_t large = rows - n * size, small_from = large * (size + 1);
        bucket = r < small_from ? 1 + r / (size + 1) : 1 + large + (r - small_from) / size;
      }
      d.out[c][i] = bucket;
    }
  }
}

// the column arrays of the C ABI -> ScanCols (checked)
int scan_cols(int64_t nrows, int ncols, const int32_t* ops, const void* const* vals, const uint8_t* const* valid,
              void* const* out_vals, int64_t* const* out_count, ScanCols* a) {
  FB_CHECK(ncols >= 1 && ncols <= FB_SCAN_MAX_COLS, "ncols=%d out of range [1,%d]", ncols, FB_SCAN_MAX_COLS);
  FB_CHECK(ops != nullptr, "NULL ops");
  memset(a, 0, sizeof(*a));
  a->ncols = ncols;
  for (int c = 0; c < ncols; ++c) {
    FB_CHECK(ops[c] >= FB_AGG_SUM_F64 && ops[c] <= FB_AGG_MAX_F64, "column %d: unknown scan op %d", c, ops[c]);
    a->op[c] = ops[c];
    a->vals[c] = vals != nullptr ? vals[c] : nullptr;
    a->valid[c] = valid != nullptr ? valid[c] : nullptr;
    a->out_vals[c] = out_vals != nullptr ? out_vals[c] : nullptr;
    a->out_count[c] = out_count != nullptr ? out_count[c] : nullptr;
    FB_CHECK(nrows == 0 || ops[c] == FB_AGG_COUNT || a->vals[c] != nullptr, "column %d: op %d needs a value column", c,
             ops[c]);
  }
  return 0;
}

// The host arrays of an f64 statistics entry -> StatCols: `nin` inputs with their validity, the count and `nout`
// words out (any array may be NULL: every entry NULL)
void stat_cols(StatCols& a, int nin, const void* const* const* in, const uint8_t* const* const* valid,
               int64_t* const* out_count, int nout, void* const* const* out) {
  for (int c = 0; c < a.ncols; ++c) {
    for (int k = 0; k < nin; ++k) {
      a.in[k][c] = in[k] != nullptr ? (const double*)in[k][c] : nullptr;
      a.valid[k][c] = valid[k] != nullptr ? valid[k][c] : nullptr;
    }
    a.out_count[c] = out_count != nullptr ? out_count[c] : nullptr;
    for (int o = 0; o < nout; ++o) a.out[o][c] = out[o] != nullptr ? (double*)out[o][c] : nullptr;
  }
}

// What every segmented scan entry shares: the checks of the counts, `fill` (the columns, checked: nonzero is an
// error), the checks of segments and scratch, the device, then the scan.  `what` names ncols in its error.
template <class T, class Fill>
int segscan_entry(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int ncols,
                  const char* what, void* scratch, size_t scratch_bytes, Fill fill) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK(ncols >= 1 && ncols <= FB_SCAN_MAX_COLS, "%s=%d out of range [1,%d]", what, ncols, FB_SCAN_MAX_COLS);
  typename T::Cols a;
  memset(&a, 0, sizeof(a));
  a.ncols = ncols;
  if (fill(a) != 0) return 1;
  if (nrows == 0) return 0;
  FB_CHECK(nseg >= 1 && d_offsets != nullptr, "%lld rows need at least one segment", (long long)nrows);
  FB_CHECK(num_tiles(nrows) < (1LL << 31), "too many rows");
  const size_t need = segscan_scratch_bytes<T>(nrows, ncols);
  FB_CHECK(scratch != nullptr && scratch_bytes >= need, "scratch too small: %zu < %zu", scratch_bytes, need);
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  return run_segscan<T>((cudaStream_t)stream, false, 0, nrows, nseg, d_offsets, a, scratch);
}

}  // namespace

extern "C" size_t fb_segmented_scan_scratch_bytes(int64_t nrows, int ncols) {
  return segscan_scratch_bytes<OpScan>(nrows, ncols);
}

extern "C" int fb_segmented_scan(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                 int ncols, const int32_t* ops, const void* const* vals,
                                 const uint8_t* const* valid, void* const* out_vals, int64_t* const* out_count,
                                 void* scratch, size_t scratch_bytes) {
  return segscan_entry<OpScan>(dev, stream, nrows, nseg, d_offsets, ncols, "ncols", scratch, scratch_bytes,
                               [&](ScanCols& a) {
                                 return scan_cols(nrows, ncols, ops, vals, valid, out_vals, out_count, &a);
                               });
}

extern "C" size_t fb_segmented_moments_scratch_bytes(int64_t nrows, int ncols) {
  return segscan_scratch_bytes<MomentScan>(nrows, ncols);
}

extern "C" int fb_segmented_moments(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                    int ncols, const void* const* vals, const uint8_t* const* valid,
                                    int64_t* const* out_count, void* const* out_m2, void* scratch,
                                    size_t scratch_bytes) {
  return segscan_entry<MomentScan>(dev, stream, nrows, nseg, d_offsets, ncols, "ncols", scratch, scratch_bytes,
                                   [&](StatCols& a) {
                                     const void* const* in[1] = {vals};
                                     const uint8_t* const* vin[1] = {valid};
                                     void* const* out[1] = {out_m2};
                                     stat_cols(a, 1, in, vin, out_count, 1, out);
                                     for (int c = 0; c < ncols; ++c)
                                       FB_CHECK(nrows == 0 || a.in[0][c] != nullptr,
                                                "column %d needs a value column", c);
                                     return 0;
                                   });
}

extern "C" size_t fb_segmented_comoments_scratch_bytes(int64_t nrows, int npairs) {
  return segscan_scratch_bytes<CoMomentScan>(nrows, npairs);
}

extern "C" int fb_segmented_comoments(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                      int npairs, const void* const* xs, const uint8_t* const* x_valid,
                                      const void* const* ys, const uint8_t* const* y_valid, int64_t* const* out_count,
                                      void* const* out_mean_x, void* const* out_mean_y, void* const* out_sxx,
                                      void* const* out_syy, void* const* out_sxy, void* scratch,
                                      size_t scratch_bytes) {
  return segscan_entry<CoMomentScan>(dev, stream, nrows, nseg, d_offsets, npairs, "npairs", scratch, scratch_bytes,
                                     [&](StatCols& a) {
                                       const void* const* in[2] = {xs, ys};
                                       const uint8_t* const* vin[2] = {x_valid, y_valid};
                                       void* const* out[5] = {out_mean_x, out_mean_y, out_sxx, out_syy, out_sxy};
                                       stat_cols(a, 2, in, vin, out_count, 5, out);
                                       for (int c = 0; c < npairs; ++c)
                                         FB_CHECK(nrows == 0 || (a.in[0][c] != nullptr && a.in[1][c] != nullptr),
                                                  "pair %d needs an x and a y column", c);
                                       return 0;
                                     });
}

extern "C" size_t fb_segmented_shape_moments_scratch_bytes(int64_t nrows, int ncols) {
  return segscan_scratch_bytes<ShapeScan>(nrows, ncols);
}

extern "C" int fb_segmented_shape_moments(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                          int ncols, const void* const* vals, const uint8_t* const* valid,
                                          int64_t* const* out_count, void* const* out_m2, void* const* out_m3,
                                          void* const* out_m4, void* scratch, size_t scratch_bytes) {
  return segscan_entry<ShapeScan>(dev, stream, nrows, nseg, d_offsets, ncols, "ncols", scratch, scratch_bytes,
                                  [&](StatCols& a) {
                                    const void* const* in[1] = {vals};
                                    const uint8_t* const* vin[1] = {valid};
                                    void* const* out[3] = {out_m2, out_m3, out_m4};
                                    stat_cols(a, 1, in, vin, out_count, 3, out);
                                    for (int c = 0; c < ncols; ++c)
                                      FB_CHECK(nrows == 0 || a.in[0][c] != nullptr, "column %d needs a value column",
                                               c);
                                    return 0;
                                  });
}

extern "C" size_t fb_segmented_ewm_scratch_bytes(int64_t nrows, int ncols) {
  return segscan_scratch_bytes<EwScan>(nrows, ncols);
}

extern "C" int fb_segmented_ewm(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                int ncols, const void* const* vals, const uint8_t* const* valid, const double* alpha,
                                const int32_t* adjust, const int32_t* positions, const void* const* times,
                                const double* time_scale, int64_t* const* out_count, void* const* out_mean,
                                void* const* out_w, void* const* out_w2, void* const* out_c, void* scratch,
                                size_t scratch_bytes) {
  return segscan_entry<EwScan>(dev, stream, nrows, nseg, d_offsets, ncols, "ncols", scratch, scratch_bytes,
                               [&](EwCols& a) {
                                 FB_CHECK(alpha != nullptr && adjust != nullptr && positions != nullptr,
                                          "NULL alpha, adjust or positions");
                                 void* const* outs[4] = {out_mean, out_w, out_w2, out_c};
                                 for (int c = 0; c < ncols; ++c) {
                                   const int pos = positions[c];
                                   FB_CHECK(pos >= FB_EWM_ROWS && pos <= FB_EWM_TIMES, "column %d: unknown positions %d",
                                            c, pos);
                                   FB_CHECK(alpha[c] > 0.0 && alpha[c] <= 1.0, "column %d: alpha %g not in (0, 1]", c,
                                            alpha[c]);
                                   a.x[c] = vals != nullptr ? (const double*)vals[c] : nullptr;
                                   a.valid[c] = valid != nullptr ? valid[c] : nullptr;
                                   FB_CHECK(nrows == 0 || a.x[c] != nullptr, "column %d needs a value column", c);
                                   double k = log2(1.0 - alpha[c]);
                                   if (pos == FB_EWM_TIMES) {
                                     FB_CHECK(times != nullptr && (nrows == 0 || times[c] != nullptr),
                                              "column %d: time decay needs a times column", c);
                                     FB_CHECK(time_scale != nullptr && time_scale[c] > 0.0 && isfinite(time_scale[c]),
                                              "column %d: time scale must be finite and > 0", c);
                                     a.t[c] = (const int64_t*)times[c];
                                     k = -time_scale[c];
                                   }
                                   a.op[c] = EwOp{k, alpha[c], adjust[c] != 0, pos == FB_EWM_OBSERVATIONS};
                                   a.out_count[c] = out_count != nullptr ? out_count[c] : nullptr;
                                   for (int o = 0; o < 4; ++o)
                                     a.out[o][c] = outs[o] != nullptr ? (double*)outs[o][c] : nullptr;
                                 }
                                 return 0;
                               });
}

extern "C" size_t fb_window_frame_scratch_bytes(int64_t nrows, int ncols, int64_t start, int64_t end, int flags) {
  return frame_scratch(nrows, ncols, make_frame(nrows, start, end, flags));
}

extern "C" int fb_window_frame(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                               int64_t start, int64_t end, int flags, int ncols, const int32_t* ops,
                               const void* const* vals, const uint8_t* const* valid, void* const* out_vals,
                               int64_t* const* out_count, void* scratch, size_t scratch_bytes) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK((flags & ~(FB_FRAME_UNBOUNDED_START | FB_FRAME_UNBOUNDED_END)) == 0, "unknown frame flags %d", flags);
  FB_CHECK(flags != 0 || start <= end, "frame start %lld > end %lld", (long long)start, (long long)end);
  ScanCols a;
  if (scan_cols(nrows, ncols, ops, vals, valid, out_vals, out_count, &a) != 0) return 1;
  if (nrows == 0) return 0;
  FB_CHECK(nseg >= 1 && d_offsets != nullptr, "%lld rows need at least one segment", (long long)nrows);
  FB_CHECK(num_tiles(nrows) < (1LL << 31), "too many rows");
  const Frame f = make_frame(nrows, start, end, flags);
  const size_t need = frame_scratch(nrows, ncols, f);
  FB_CHECK(need == 0 || (scratch != nullptr && scratch_bytes >= need), "scratch too small: %zu < %zu", scratch_bytes,
           need);
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (f.tile) {
    static std::mutex mu;
    static uint64_t optin_done = 0;
    {
      std::lock_guard<std::mutex> lock(mu);
      if (!(dev >= 0 && dev < 64 && ((optin_done >> dev) & 1))) {
        FB_CUDA(cudaFuncSetAttribute(fb_window_frame_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(FrameSmem)));
        if (dev >= 0 && dev < 64) optin_done |= 1ull << dev;
      }
    }
    const int64_t per_tile = kFrameSpan - (f.width - 1);
    const int64_t grid = (nrows + per_tile - 1) / per_tile;
    FB_CHECK(grid < (1LL << 31), "too many rows");
    fb_window_frame_tile_kernel<<<(unsigned)grid, kFrameThreads, sizeof(FrameSmem), st>>>(
        nrows, nseg, d_offsets, a, f.start, (int)f.width, per_tile);
    FB_CUDA(cudaGetLastError());
    return 0;
  }
  // P and / or S into scratch, then the combine pass
  const bool need_p = f.flags != FB_FRAME_UNBOUNDED_END;                 // bounded, (None, e), (None, None)
  const bool need_s = f.flags == 0 || f.flags == FB_FRAME_UNBOUNDED_END;  // bounded, (s, None)
  char* tiles = (char*)scratch;
  char* sides = tiles + align256(segscan_scratch_bytes<OpScan>(nrows, ncols));
  const size_t side = (size_t)ncols * (size_t)nrows;
  uint64_t* pv = need_p ? (uint64_t*)sides : nullptr;
  int64_t* pc = need_p ? (int64_t*)(pv + side) : nullptr;
  uint64_t* sv = need_s ? (uint64_t*)(need_p ? (char*)sides + 16 * side : sides) : nullptr;
  int64_t* sc = need_s ? (int64_t*)(sv + side) : nullptr;
  ScanCols b = a;
  if (need_p) {
    for (int c = 0; c < ncols; ++c) {
      b.out_vals[c] = pv + c * nrows;
      b.out_count[c] = pc + c * nrows;
    }
    if (run_segscan<OpScan>(st, false, f.width, nrows, nseg, d_offsets, b, tiles) != 0) return 2;
  }
  if (need_s) {
    for (int c = 0; c < ncols; ++c) {
      b.out_vals[c] = sv + c * nrows;
      b.out_count[c] = sc + c * nrows;
    }
    if (run_segscan<OpScan>(st, true, f.width, nrows, nseg, d_offsets, b, tiles) != 0) return 2;
  }
  fb_window_frame_combine_kernel<<<(unsigned)num_tiles(nrows), kThreads, 0, st>>>(
      nrows, nseg, d_offsets, a, f.start, f.end, f.flags, f.width, pv, pc, sv, sc);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" size_t fb_window_range_bounds_scratch_bytes(int64_t nseg) {
  return nseg > 0 ? (size_t)nseg * sizeof(int64_t) : 0;
}

extern "C" int fb_window_range_bounds(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                      const void* d_keys, const uint8_t* d_key_valid, int key_class, int descending,
                                      uint64_t start, uint64_t end, int flags, int64_t* d_lo, int64_t* d_hi,
                                      void* scratch, size_t scratch_bytes) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK((flags & ~(FB_FRAME_UNBOUNDED_START | FB_FRAME_UNBOUNDED_END)) == 0, "unknown frame flags %d", flags);
  FB_CHECK(key_class == FB_RANGE_KEY_I64 || key_class == FB_RANGE_KEY_U64 || key_class == FB_RANGE_KEY_F64,
           "unknown key class %d", key_class);
  if (nrows == 0) return 0;
  FB_CHECK(nseg >= 1 && d_offsets != nullptr, "%lld rows need at least one segment", (long long)nrows);
  FB_CHECK(d_keys != nullptr && d_lo != nullptr && d_hi != nullptr, "NULL keys or outputs");
  FB_CHECK(scratch != nullptr && scratch_bytes >= fb_window_range_bounds_scratch_bytes(nseg),
           "scratch too small: %zu < %zu", scratch_bytes, fb_window_range_bounds_scratch_bytes(nseg));
  const int64_t grid = (nrows + kRangeThreads - 1) / kRangeThreads;
  FB_CHECK(grid < (1LL << 31), "too many rows");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* null_start = (int64_t*)scratch;
  fb_range_null_start_kernel<<<(unsigned)((nseg + kRangeThreads - 1) / kRangeThreads), kRangeThreads, 0, st>>>(
      nseg, d_offsets, d_key_valid, null_start);
  FB_CUDA(cudaGetLastError());
  fb_range_bounds_kernel<<<(unsigned)grid, kRangeThreads, 0, st>>>(nrows, nseg, d_offsets, null_start,
                                                                    (const uint64_t*)d_keys, key_class, descending,
                                                                    start, end, flags, d_lo, d_hi);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" size_t fb_window_bounded_scratch_bytes(int64_t nrows, int ncols) {
  if (nrows <= 0 || ncols <= 0) return 0;
  return (size_t)tree_levels(nrows).total * 16 * (size_t)ncols;
}

extern "C" int fb_window_bounded(int dev, void* stream, int64_t nrows, const int64_t* d_lo, const int64_t* d_hi,
                                 int ncols, const int32_t* ops, const void* const* vals, const uint8_t* const* valid,
                                 void* const* out_vals, int64_t* const* out_count, void* scratch,
                                 size_t scratch_bytes) {
  FB_CHECK(nrows >= 0, "negative row count");
  ScanCols a;
  if (scan_cols(nrows, ncols, ops, vals, valid, out_vals, out_count, &a) != 0) return 1;
  if (nrows == 0) return 0;
  FB_CHECK(d_lo != nullptr && d_hi != nullptr, "NULL bounds");
  const int64_t grid = (nrows + kThreads - 1) / kThreads;
  FB_CHECK(grid < (1LL << 31), "too many rows");
  const size_t need = fb_window_bounded_scratch_bytes(nrows, ncols);
  FB_CHECK(need == 0 || (scratch != nullptr && scratch_bytes >= need), "scratch too small: %zu < %zu", scratch_bytes,
           need);
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (build_tree(dev, st, a, nrows, scratch) != 0) return 2;
  const TreeLevels L = tree_levels(nrows);
  const uint64_t* tv = (const uint64_t*)scratch;
  fb_tree_query_kernel<<<(unsigned)grid, kThreads, 0, st>>>(a, L, nrows, d_lo, d_hi, tv,
                                                             (const int64_t*)(tv + (size_t)ncols * L.total));
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_window_tree(int dev, void* stream, int64_t nrows, int ncols, const int32_t* ops,
                              const void* const* vals, const uint8_t* const* valid, void* scratch,
                              size_t scratch_bytes) {
  FB_CHECK(nrows >= 0, "negative row count");
  ScanCols a;
  if (scan_cols(nrows, ncols, ops, vals, valid, nullptr, nullptr, &a) != 0) return 1;
  if (nrows == 0) return 0;
  const size_t need = fb_window_bounded_scratch_bytes(nrows, ncols);
  FB_CHECK(need == 0 || (scratch != nullptr && scratch_bytes >= need), "scratch too small: %zu < %zu", scratch_bytes,
           need);
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  return build_tree(dev, (cudaStream_t)stream, a, nrows, scratch) != 0 ? 2 : 0;
}

extern "C" int fb_window_value(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                               int64_t start, int64_t end, int flags, const int64_t* d_lo, const int64_t* d_hi,
                               int ncols, const int64_t* nths, const int32_t* widths, const void* const* vals,
                               const uint8_t* const* valid, void* const* out_vals, uint8_t* const* out_valid) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK((flags & ~(FB_FRAME_UNBOUNDED_START | FB_FRAME_UNBOUNDED_END)) == 0, "unknown frame flags %d", flags);
  FB_CHECK((d_lo == nullptr) == (d_hi == nullptr), "give both of d_lo / d_hi or neither");
  FB_CHECK(ncols >= 1 && ncols <= FB_SCAN_MAX_COLS, "ncols=%d out of range [1,%d]", ncols, FB_SCAN_MAX_COLS);
  FB_CHECK(nths != nullptr && widths != nullptr && vals != nullptr && out_vals != nullptr && out_valid != nullptr,
           "NULL column arrays");
  ValueCols a;
  memset(&a, 0, sizeof(a));
  a.ncols = ncols;
  for (int c = 0; c < ncols; ++c) {
    FB_CHECK(nths[c] == FB_VALUE_LAST || nths[c] >= 1, "column %d: nth %lld < 1", c, (long long)nths[c]);
    FB_CHECK(widths[c] == 1 || widths[c] == 2 || widths[c] == 4 || widths[c] == 8, "column %d: width %d", c,
             widths[c]);
    a.nth[c] = nths[c] > nrows ? nrows + 1 : nths[c];  // past every frame either way; lo + n - 1 cannot wrap
    a.width[c] = widths[c];
    a.vals[c] = vals[c];
    a.valid[c] = valid != nullptr ? valid[c] : nullptr;
    a.out[c] = out_vals[c];
    a.out_valid[c] = out_valid[c];
    FB_CHECK(nrows == 0 || (a.vals[c] != nullptr && a.out[c] != nullptr && a.out_valid[c] != nullptr),
             "column %d: NULL values or outputs", c);
  }
  if (nrows == 0) return 0;
  FB_CHECK(d_lo != nullptr || (nseg >= 1 && d_offsets != nullptr), "%lld rows need at least one segment",
           (long long)nrows);
  if (d_lo == nullptr) FB_CHECK(flags != 0 || start <= end, "frame start %lld > end %lld", (long long)start,
                                (long long)end);
  const Frame f = make_frame(nrows, start, end, flags);
  const int64_t grid = (nrows + kRangeThreads - 1) / kRangeThreads;
  FB_CHECK(grid < (1LL << 31), "too many rows");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_window_value_kernel<<<(unsigned)grid, kRangeThreads, 0, (cudaStream_t)stream>>>(
      nrows, nseg, d_offsets, f.start, f.end, f.flags, d_lo, d_hi, a);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" size_t fb_window_distribution_scratch_bytes(int64_t nrows) {
  return nrows > 0 ? 2 * sizeof(int64_t) * (size_t)num_tiles(nrows) : 0;
}

extern "C" int fb_window_distribution(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                                      const uint8_t* d_heads, double* d_percent_rank, double* d_cume_dist,
                                      int nntile, const int64_t* ntiles, int64_t* const* d_ntile, void* scratch,
                                      size_t scratch_bytes) {
  FB_CHECK(nrows >= 0 && nseg >= 0, "negative row or segment count");
  FB_CHECK(nntile >= 0 && nntile <= FB_SCAN_MAX_COLS, "nntile=%d out of range [0,%d]", nntile, FB_SCAN_MAX_COLS);
  DistCols d;
  memset(&d, 0, sizeof(d));
  d.ncols = nntile;
  for (int c = 0; c < nntile; ++c) {
    FB_CHECK(ntiles != nullptr && d_ntile != nullptr, "NULL NTILE arrays");
    FB_CHECK(ntiles[c] >= 1, "NTILE %d: n = %lld < 1", c, (long long)ntiles[c]);
    FB_CHECK(nrows == 0 || d_ntile[c] != nullptr, "NTILE %d: NULL output", c);
    d.n[c] = ntiles[c];
    d.out[c] = d_ntile[c];
  }
  if (nrows == 0) return 0;
  FB_CHECK(nseg >= 1 && d_offsets != nullptr && d_heads != nullptr, "%lld rows need segments and head bytes",
           (long long)nrows);
  const int64_t tiles = num_tiles(nrows);
  FB_CHECK(tiles < (1LL << 31), "too many rows");
  FB_CHECK(scratch != nullptr && scratch_bytes >= fb_window_distribution_scratch_bytes(nrows),
           "scratch too small: %zu < %zu", scratch_bytes, fb_window_distribution_scratch_bytes(nrows));
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* tile_first = (int64_t*)scratch;
  int64_t* tile_last = tile_first + tiles;
  fb_peer_tile_kernel<<<(unsigned)tiles, kThreads, 0, st>>>(nrows, d_heads, tile_first, tile_last);
  FB_CUDA(cudaGetLastError());
  fb_peer_carry_kernel<<<1, kCarryThreads, 0, st>>>(tiles, tile_first, tile_last);
  FB_CUDA(cudaGetLastError());
  fb_window_distribution_kernel<<<(unsigned)tiles, kThreads, 0, st>>>(nrows, nseg, d_offsets, d_heads, tile_first,
                                                                       tile_last, d_percent_rank, d_cume_dist, d);
  FB_CUDA(cudaGetLastError());
  return 0;
}
