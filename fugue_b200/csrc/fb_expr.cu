// Column-expression evaluator for sm_90a: one pass over HBM per SELECT list.
//
// ExecutionEngine.select / filter / assign (fugue/execution/execution_engine.py:736-887) evaluate
// expression trees (fugue/column/expressions.py); the reference turns them into SQL text and hands
// them to qpd/pandas, which materialises one temporary column per operator.  Here the host compiles
// the whole SELECT list (or WHERE predicate) into one short accumulator-machine program:
//
//   * a thread owns kExprItems rows; the accumulator (their current values + a validity bit each)
//     sits in hardware registers for the whole program;
//   * the second operand of an instruction is fetched straight from its source: a column in HBM
//     (coalesced, converted from its storage type on the fly), an immediate, or a temporary in
//     shared memory - temporaries are only needed when both sides of an operator are compound, so
//     typical expressions never touch shared memory (a first version that kept every intermediate
//     in shared-memory vector registers was bound by shared-memory wavefronts);
//   * the interpreter dispatches once per instruction per thread and then runs its rows unrolled,
//     so the switch is amortised; every output is written by its own FB_X_OUT instruction;
//   * SQL NULL semantics: arithmetic and comparisons propagate NULL (validity bits are ANDed for
//     all rows of the thread at once), AND / OR are Kleene three-valued, IS NULL / IS NOT NULL /
//     COALESCE read the validity bits;
//   * CASE runs without branching: every branch is computed for every row and FB_X_SEL keeps, per row,
//     the value of the first branch whose condition is TRUE.  No op traps (x % 0 is NULL, not a fault),
//     so computing a branch a row does not take is harmless.
#include <mutex>

#include <cuda_fp16.h>

#include "fb_calendar.cuh"

namespace {

constexpr int kExprThreads = 256;
constexpr int kExprItems = 8;
constexpr int kExprTile = kExprThreads * kExprItems;
constexpr unsigned kAllValid = (1u << kExprItems) - 1;

struct ExprProgram {
  const void* col_ptr[FB_EXPR_MAX_COLS];
  const uint8_t* col_valid[FB_EXPR_MAX_COLS];
  int32_t col_type[FB_EXPR_MAX_COLS];
  void* out_ptr[FB_EXPR_MAX_OUTS];
  uint8_t* out_valid[FB_EXPR_MAX_OUTS];
  int32_t out_type[FB_EXPR_MAX_OUTS];
  int32_t nins;
  fb_expr_ins ins[FB_EXPR_MAX_INS];
};
static_assert(sizeof(ExprProgram) <= 4000, "program must fit the kernel parameter space");

__device__ __forceinline__ double as_f(uint64_t b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ uint64_t f_bits(double d) { return (uint64_t)__double_as_longlong(d); }

template <typename T, bool kFloat, bool kFull>
__device__ __forceinline__ void load_col(const void* p, int64_t row0, int tid, int nk, uint64_t (&v)[kExprItems]) {
  const T* __restrict__ q = (const T*)p + row0;
#pragma unroll
  for (int k = 0; k < kExprItems; ++k) {
    const int i = k * kExprThreads + tid;
    if (kFull || i < nk) {
      if (kFloat) v[k] = f_bits((double)q[i]);
      else v[k] = (uint64_t)(int64_t)q[i];  // unsigned T zero-extends, signed T sign-extends
    }
  }
}

// float16 is stored as its 16 bits; every half value is exact in a double
template <bool kFull>
__device__ __forceinline__ void load_f16(const void* p, int64_t row0, int tid, int nk, uint64_t (&v)[kExprItems]) {
  const __half* __restrict__ q = (const __half*)p + row0;
#pragma unroll
  for (int k = 0; k < kExprItems; ++k) {
    const int i = k * kExprThreads + tid;
    if (kFull || i < nk) v[k] = f_bits((double)__half2float(q[i]));
  }
}

template <typename T, bool kFloat, bool kFull>
__device__ __forceinline__ void store_col(void* p, int64_t row0, int tid, int nk, const uint64_t (&v)[kExprItems],
                                          unsigned valid) {
  T* __restrict__ q = (T*)p + row0;
#pragma unroll
  for (int k = 0; k < kExprItems; ++k) {
    const int i = k * kExprThreads + tid;
    if (kFull || i < nk) {
      const uint64_t bits = (valid >> k) & 1u ? v[k] : 0ull;  // NULL rows store 0
      if (kFloat) q[i] = (T)as_f(bits);
      else q[i] = (T)(int64_t)bits;
    }
  }
}

template <bool kFull>
__device__ __forceinline__ void store_f16(void* p, int64_t row0, int tid, int nk, const uint64_t (&v)[kExprItems],
                                          unsigned valid) {
  __half* __restrict__ q = (__half*)p + row0;
#pragma unroll
  for (int k = 0; k < kExprItems; ++k) {
    const int i = k * kExprThreads + tid;
    if (kFull || i < nk) q[i] = __double2half(as_f((valid >> k) & 1u ? v[k] : 0ull));  // one rounding, to nearest even
  }
}

// FB_X_LOOKUP: acc <- table[acc] (8-byte entries) for the valid rows whose entry number is in [0, nent); every
// other row is NULL
__device__ __forceinline__ void lookup(const uint64_t* __restrict__ q, const uint8_t* m, uint64_t nent,
                                       uint64_t (&acc)[kExprItems], unsigned& accv) {
  unsigned nv = 0;
#pragma unroll
  for (int k = 0; k < kExprItems; ++k) {
    const uint64_t e = acc[k];
    acc[k] = 0;
    if (((accv >> k) & 1u) && e < nent) {  // a NULL row's stored code means nothing: never an index
      acc[k] = q[e];
      if (m == nullptr || m[e] != 0) nv |= 1u << k;
    }
  }
  accv = nv;
}

// ---- scalar functions (one row).  An integer is int64 and wraps; a float is float64.
__device__ __forceinline__ bool mod_i(const uint64_t x, const uint64_t y, uint64_t& r) {  // false: NULL (y = 0)
  const int64_t a = (int64_t)x, b = (int64_t)y;
  r = (b == -1 || b == 0) ? 0 : (uint64_t)(a % b);  // INT64_MIN % -1 would trap: every x % -1 is 0
  return b != 0;
}

// fmod is exact.  y = +-0.0 is NULL even for a NaN x; fmod(+-inf, y) is a domain error (NaN from non-NaN)
__device__ __noinline__ double fn_fmod(double x, double y) { return fmod(x, y); }

__device__ __forceinline__ bool mod_f(const uint64_t xb, const uint64_t yb, uint64_t& rb) {
  const double x = as_f(xb), y = as_f(yb), r = fn_fmod(x, y);
  rb = f_bits(r);
  return y != 0.0 && !(isnan(r) && !isnan(x) && !isnan(y));
}

__device__ __forceinline__ double pow10_f(int e) {  // 10^e for e in [0, 18]: every one is exact in a double
  double p = 1.0;
  for (int i = 0; i < e; ++i) p *= 10.0;  // each product is an integer below 2^63 with at most 53 significant bits
  return p;
}

// ROUND(x, d): d = 0 is C round; else DuckDB's round(x * 10^d) / 10^d, and x itself when the scaled value is not finite
__device__ __forceinline__ double round_f(double x, int d) {
  if (d == 0) return round(x);
  const double p = pow10_f(d < 0 ? -d : d);
  const double s = d > 0 ? x * p : x / p;
  if (!isfinite(s)) return x;
  return d > 0 ? round(s) / p : round(s) * p;
}

// ROUND(x, d) of an int64, d < 0: the nearest multiple of 10^-d, half away from zero; wraps like + - *
__device__ __forceinline__ uint64_t round_i(uint64_t x, int d) {
  int64_t p = 1;
  for (int i = 0; i < -d; ++i) p *= 10;
  const int64_t a = (int64_t)x, r = a % p;
  uint64_t q = x - (uint64_t)r;
  const uint64_t ar = (uint64_t)(r < 0 ? -r : r);
  if (2 * ar >= (uint64_t)p) q += a < 0 ? (uint64_t)(-p) : (uint64_t)p;
  return q;
}

// IEEE totalOrder as a signed key: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN (aggregate MIN / MAX)
__device__ __forceinline__ int64_t total_key(uint64_t b) {
  const int64_t s = (int64_t)b;
  return s >= 0 ? s : s ^ 0x7FFFFFFFFFFFFFFFll;
}

// the transcendental functions run out of line, once per row: inlined into the 8-row unrolled loop they cost registers
__device__ __noinline__ double fn_exp(double x) { return exp(x); }
__device__ __noinline__ double fn_ln(double x) { return log(x); }
__device__ __noinline__ double fn_log10(double x) { return log10(x); }
__device__ __noinline__ double fn_pow(double x, double y) { return pow(x, y); }

// ---- temporal ops (one row): proleptic Gregorian calendar (fb_calendar.cuh), UTC, no leap seconds.  A value is an
// int64 count of `unit`s since 1970-01-01 00:00.
__device__ __forceinline__ int64_t units_per_second(int unit) {
  switch (unit) {
    case FB_TU_MS: return 1000ll;
    case FB_TU_US: return 1000000ll;
    case FB_TU_NS: return 1000000000ll;
    default: return 1ll;
  }
}

// x -> whole days since the epoch and the second of that day (0 for a date)
__device__ __forceinline__ void split_days(int64_t x, int unit, int64_t& days, int64_t& sod) {
  int64_t s = x;
  switch (unit) {
    case FB_TU_DAY: days = x; sod = 0; return;
    case FB_TU_MS: s = fdiv<1000ll>(x); break;
    case FB_TU_US: s = fdiv<1000000ll>(x); break;
    case FB_TU_NS: s = fdiv<1000000000ll>(x); break;
    default: break;
  }
  days = fdiv<86400ll>(s);
  sod = s - days * 86400ll;
}

__device__ __forceinline__ int64_t join_days(int64_t days, int64_t sod, int unit) {
  if (unit == FB_TU_DAY) return days;
  return wmul(wadd(wmul(days, 86400ll), sod), units_per_second(unit));
}

// days since the epoch -> year, month (1-12), day (1-31), day of the year (1-366): 400-year eras of 146 097 days,
// years that start on March 1
__device__ __forceinline__ void civil_from_days(int64_t days, int64_t& y, int& m, int& d, int& doy) {
  const int64_t z = wadd(days, 719468ll);
  const int64_t era = fdiv<146097ll>(z);
  const int doe = (int)(z - era * 146097ll);                                    // [0, 146096]
  const int yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;        // [0, 399]
  const int doy_m = doe - (365 * yoe + yoe / 4 - yoe / 100);                    // [0, 365], from March 1
  const int mp = (5 * doy_m + 2) / 153;                                         // [0, 11]
  d = doy_m - (153 * mp + 2) / 5 + 1;
  m = mp < 10 ? mp + 3 : mp - 9;
  y = wadd(wadd((int64_t)yoe, wmul(era, 400ll)), (int64_t)(m <= 2));
  doy = mp < 10 ? doy_m + 60 + (int)is_leap(y) : doy_m - 305;
}

__device__ __forceinline__ int iso_weekday(int64_t days) {  // 1 = Monday ... 7 = Sunday; 1970-01-01 was a Thursday
  const int64_t t = wadd(days, 3ll);
  return (int)(t - fdiv<7ll>(t) * 7ll) + 1;
}

__device__ __forceinline__ uint64_t ts_part(int64_t x, int field, int unit) {
  int64_t days, sod, y;
  int m, d, doy;
  split_days(x, unit, days, sod);
  switch (field) {
    case FB_TF_HOUR: return (uint64_t)(sod / 3600);
    case FB_TF_MINUTE: return (uint64_t)(sod / 60 % 60);
    case FB_TF_SECOND: return (uint64_t)(sod % 60);
    case FB_TF_DOW: return (uint64_t)(iso_weekday(days) % 7);
    case FB_TF_ISODOW: return (uint64_t)iso_weekday(days);
    case FB_TF_WEEK:
    case FB_TF_ISOYEAR: days = wadd(days, (int64_t)(4 - iso_weekday(days))); break;  // the Thursday of the ISO week
    default: break;
  }
  civil_from_days(days, y, m, d, doy);
  switch (field) {
    case FB_TF_MONTH: return (uint64_t)m;
    case FB_TF_DAY: return (uint64_t)d;
    case FB_TF_QUARTER: return (uint64_t)((m - 1) / 3 + 1);
    case FB_TF_DOY: return (uint64_t)doy;
    case FB_TF_WEEK: return (uint64_t)((doy - 1) / 7 + 1);
    default: return (uint64_t)y;  // FB_TF_YEAR, FB_TF_ISOYEAR
  }
}

__device__ __forceinline__ uint64_t ts_trunc(int64_t x, int part, int unit) {
  int64_t days, sod, y;
  int m, d, doy;
  split_days(x, unit, days, sod);
  switch (part) {
    case FB_TP_SECOND: break;
    case FB_TP_MINUTE: sod -= sod % 60; break;
    case FB_TP_HOUR: sod -= sod % 3600; break;
    case FB_TP_DAY: sod = 0; break;
    case FB_TP_WEEK: sod = 0; days = wsub(days, (int64_t)(iso_weekday(days) - 1)); break;
    default:
      civil_from_days(days, y, m, d, doy);
      sod = 0;
      days = days_from_civil(y, part == FB_TP_YEAR ? 1 : part == FB_TP_QUARTER ? (m - 1) / 3 * 3 + 1 : m, 1);
      break;
  }
  return (uint64_t)join_days(days, sod, unit);
}

// whole parts since 1970-01-01 00:00 (weeks: since Monday 1969-12-29)
__device__ __forceinline__ uint64_t ts_index(int64_t x, int part, int unit) {
  int64_t days, sod, y;
  int m, d, doy;
  split_days(x, unit, days, sod);
  switch (part) {
    case FB_TP_SECOND: return (uint64_t)wadd(wmul(days, 86400ll), sod);
    case FB_TP_MINUTE: return (uint64_t)wadd(wmul(days, 1440ll), sod / 60);
    case FB_TP_HOUR: return (uint64_t)wadd(wmul(days, 24ll), sod / 3600);
    case FB_TP_DAY: return (uint64_t)days;
    case FB_TP_WEEK: return (uint64_t)fdiv<7ll>(wadd(days, 3ll));
    default: break;
  }
  civil_from_days(days, y, m, d, doy);
  y = wsub(y, 1970ll);
  if (part == FB_TP_YEAR) return (uint64_t)y;
  if (part == FB_TP_QUARTER) return (uint64_t)wadd(wmul(y, 4ll), (int64_t)((m - 1) / 3));
  return (uint64_t)wadd(wmul(y, 12ll), (int64_t)(m - 1));
}

// x + n calendar months: the day of the month clamped to the target month's last day, the time of day kept
__device__ __forceinline__ uint64_t ts_addmon(int64_t x, int64_t n, int unit) {
  int64_t days, sod, y;
  int m, d, doy;
  split_days(x, unit, days, sod);
  const int64_t sub = wsub(x, join_days(days, sod, unit));  // the fraction of a second, in units
  civil_from_days(days, y, m, d, doy);
  const int64_t mi = wadd(wadd(wmul(y, 12ll), (int64_t)(m - 1)), n);
  const int64_t y2 = fdiv<12ll>(mi);
  const int m2 = (int)(mi - y2 * 12ll) + 1;
  const int last = m2 == 2 ? 28 + (int)is_leap(y2) : 30 + ((m2 + (m2 >> 3)) & 1);
  return (uint64_t)wadd(join_days(days_from_civil(y2, m2, d < last ? d : last), sod, unit), sub);
}

__device__ __forceinline__ uint64_t mulsat_i(int64_t x, int64_t b) {  // b >= 1
  const int64_t lo = wmul(x, b);
  if (__mul64hi(x, b) != (lo >> 63)) return x < 0 ? 0x8000000000000000ull : 0x7FFFFFFFFFFFFFFFull;
  return (uint64_t)lo;
}

__device__ __forceinline__ uint64_t floordiv_i(int64_t x, int64_t b) {  // b >= 1 (checked on the host)
  const int64_t q = x / b;
  return (uint64_t)(q - (int64_t)(x % b < 0));
}

// the temporal ops run out of line, once per row, like the transcendental functions below: the interpreter's switch
// and its registers stay what they were.  `code`: field or part | unit << 8
__device__ __noinline__ uint64_t fn_mulsat(uint64_t x, uint64_t b) { return mulsat_i((int64_t)x, (int64_t)b); }
__device__ __noinline__ uint64_t fn_floordiv(uint64_t x, uint64_t b) { return floordiv_i((int64_t)x, (int64_t)b); }
__device__ __noinline__ uint64_t fn_ts_part(uint64_t x, int code) { return ts_part((int64_t)x, code & 0xFF, code >> 8); }
__device__ __noinline__ uint64_t fn_ts_trunc(uint64_t x, int code) { return ts_trunc((int64_t)x, code & 0xFF, code >> 8); }
__device__ __noinline__ uint64_t fn_ts_index(uint64_t x, int code) { return ts_index((int64_t)x, code & 0xFF, code >> 8); }
__device__ __noinline__ uint64_t fn_ts_addmon(uint64_t x, uint64_t n, int unit) {
  return ts_addmon((int64_t)x, (int64_t)n, unit);
}

// one tile of kExprTile rows (kFull: no bounds checks; only the last tile of a table is partial)
template <bool kFull>
__device__ __forceinline__ void run_tile(const ExprProgram& P, int64_t row0, int nk, int tid, uint64_t* tmp_v,
                                         uint8_t* tmp_m) {
  {
    uint64_t acc[kExprItems];
    unsigned accv = kAllValid;
#pragma unroll
    for (int k = 0; k < kExprItems; ++k) acc[k] = 0;
    for (int pc = 0; pc < P.nins; ++pc) {
      const fb_expr_ins in = P.ins[pc];
      // ---- operand B
      uint64_t b[kExprItems];
      unsigned bv = kAllValid;
      if (in.kind == FB_XK_IMM) {
#pragma unroll
        for (int k = 0; k < kExprItems; ++k) b[k] = (uint64_t)in.imm;
      } else if (in.kind == FB_XK_COL && in.op != FB_X_LOOKUP) {  // a lookup table is indexed by acc
        const void* p = P.col_ptr[in.b];
        switch (P.col_type[in.b]) {
          case FB_T_I8: load_col<int8_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_I16: load_col<int16_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_I32: load_col<int32_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_I64: load_col<int64_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_U8: load_col<uint8_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_F32: load_col<float, true, kFull>(p, row0, tid, nk, b); break;
          case FB_T_U16: load_col<uint16_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_U32: load_col<uint32_t, false, kFull>(p, row0, tid, nk, b); break;
          case FB_T_F16: load_f16<kFull>(p, row0, tid, nk, b); break;
          default: load_col<int64_t, false, kFull>(p, row0, tid, nk, b); break;  // FB_T_F64: raw bits
        }
        const uint8_t* m = P.col_valid[in.b];
        if (m != nullptr) {
          bv = 0;
#pragma unroll
          for (int k = 0; k < kExprItems; ++k) {
            const int i = k * kExprThreads + tid;
            if ((kFull || i < nk) && m[row0 + i] != 0) bv |= 1u << k;
          }
        }
      } else if (in.kind == FB_XK_REG) {
        const uint64_t* r = tmp_v + (size_t)in.b * kExprTile;
#pragma unroll
        for (int k = 0; k < kExprItems; ++k) b[k] = r[k * kExprThreads + tid];
        bv = tmp_m[in.b * kExprThreads + tid];
      } else if (in.kind == FB_XK_NULL) {
        bv = 0;
      }
      if (in.kind == FB_XK_NONE || in.kind == FB_XK_NULL || (!kFull && in.kind == FB_XK_COL)) {
#pragma unroll
        for (int k = 0; k < kExprItems; ++k)  // defined values for lanes that were not loaded
          if (in.kind != FB_XK_COL || k * kExprThreads + tid >= nk) b[k] = 0;
      }
      if (in.flags & FB_XF_B_I2F) {
#pragma unroll
        for (int k = 0; k < kExprItems; ++k) b[k] = f_bits((double)(int64_t)b[k]);
      }
#define FB_ROWS(...) _Pragma("unroll") for (int k = 0; k < kExprItems; ++k) { __VA_ARGS__ }
#define FB_BIN(EXPR) FB_ROWS(const uint64_t x = acc[k], y = b[k]; acc[k] = (EXPR);) accv &= bv;
#define FB_UN(EXPR) FB_ROWS(const uint64_t x = acc[k]; acc[k] = (EXPR);)
// CHK: a binary op whose call is false where the row becomes NULL; FUN / FBIN: float functions under the domain rule
#define FB_CHK(CALL) { unsigned ok = 0; FB_ROWS(if (CALL) ok |= 1u << k;) accv &= bv & ok; }
#define FB_FUN(EXPR) { unsigned bad = 0; FB_ROWS(const double x = as_f(acc[k]); const double r = (EXPR); \
                       acc[k] = f_bits(r); if (isnan(r) && !isnan(x)) bad |= 1u << k;) accv &= ~bad; }
#define FB_FBIN(EXPR) { unsigned bad = 0; FB_ROWS(const double x = as_f(acc[k]), y = as_f(b[k]); const double r = (EXPR); \
                        acc[k] = f_bits(r); if (isnan(r) && !isnan(x) && !isnan(y)) bad |= 1u << k;) accv &= bv & ~bad; }
      switch (in.op) {
        case FB_X_MOV: FB_ROWS(acc[k] = b[k];) accv = bv; break;
        case FB_X_ST: {
          uint64_t* r = tmp_v + (size_t)in.b * kExprTile;
          FB_ROWS(r[k * kExprThreads + tid] = acc[k];)
          tmp_m[in.b * kExprThreads + tid] = (uint8_t)accv;
          break;
        }
        case FB_X_OUT: {
          void* p = P.out_ptr[in.b];
          switch (P.out_type[in.b]) {
            case FB_T_I8: store_col<int8_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_I16: store_col<int16_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_I32: store_col<int32_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_I64: store_col<int64_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_U8: store_col<uint8_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_F32: store_col<float, true, kFull>(p, row0, tid, nk, acc, accv); break;
            // unsigned stores keep the low bits, exactly as the signed stores of the same width do
            case FB_T_U16: store_col<int16_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_U32: store_col<int32_t, false, kFull>(p, row0, tid, nk, acc, accv); break;
            case FB_T_F16: store_f16<kFull>(p, row0, tid, nk, acc, accv); break;
            default: store_col<int64_t, false, kFull>(p, row0, tid, nk, acc, accv); break;  // FB_T_F64
          }
          uint8_t* m = P.out_valid[in.b];
          if (m != nullptr) {
            FB_ROWS(const int i = k * kExprThreads + tid;
                    if (kFull || i < nk) m[row0 + i] = (uint8_t)((accv >> k) & 1u);)
          }
          break;
        }
        case FB_X_I2F: FB_UN(f_bits((double)(int64_t)x)) break;
        case FB_X_F2I: FB_UN((uint64_t)(int64_t)as_f(x)) break;
        case FB_X_NEG_I: FB_UN(0 - x) break;
        case FB_X_NEG_F: FB_UN(x ^ 0x8000000000000000ull) break;
        case FB_X_NOT: FB_UN((uint64_t)(x == 0)) break;
        case FB_X_IS_NULL: FB_ROWS(acc[k] = (uint64_t)(((accv >> k) & 1u) == 0);) accv = kAllValid; break;
        case FB_X_NOT_NULL: FB_ROWS(acc[k] = (uint64_t)((accv >> k) & 1u);) accv = kAllValid; break;
        case FB_X_TOBOOL_I: FB_UN((uint64_t)(x != 0)) break;
        case FB_X_TOBOOL_F: FB_UN((uint64_t)(as_f(x) != 0.0)) break;
        case FB_X_ADD_I: FB_BIN(x + y) break;
        case FB_X_SUB_I: FB_BIN(x - y) break;
        case FB_X_RSUB_I: FB_BIN(y - x) break;
        case FB_X_MUL_I: FB_BIN(x * y) break;
        case FB_X_ADD_F: FB_BIN(f_bits(as_f(x) + as_f(y))) break;
        case FB_X_SUB_F: FB_BIN(f_bits(as_f(x) - as_f(y))) break;
        case FB_X_RSUB_F: FB_BIN(f_bits(as_f(y) - as_f(x))) break;
        case FB_X_MUL_F: FB_BIN(f_bits(as_f(x) * as_f(y))) break;
        case FB_X_DIV_F: FB_BIN(f_bits(as_f(x) / as_f(y))) break;
        case FB_X_RDIV_F: FB_BIN(f_bits(as_f(y) / as_f(x))) break;
        case FB_X_LT_I: FB_BIN((uint64_t)((int64_t)x < (int64_t)y)) break;
        case FB_X_LE_I: FB_BIN((uint64_t)((int64_t)x <= (int64_t)y)) break;
        case FB_X_GT_I: FB_BIN((uint64_t)((int64_t)x > (int64_t)y)) break;
        case FB_X_GE_I: FB_BIN((uint64_t)((int64_t)x >= (int64_t)y)) break;
        case FB_X_EQ_I: FB_BIN((uint64_t)(x == y)) break;
        case FB_X_NE_I: FB_BIN((uint64_t)(x != y)) break;
        case FB_X_LT_F: FB_BIN((uint64_t)(as_f(x) < as_f(y))) break;
        case FB_X_LE_F: FB_BIN((uint64_t)(as_f(x) <= as_f(y))) break;
        case FB_X_GT_F: FB_BIN((uint64_t)(as_f(x) > as_f(y))) break;
        case FB_X_GE_F: FB_BIN((uint64_t)(as_f(x) >= as_f(y))) break;
        case FB_X_EQ_F: FB_BIN((uint64_t)(as_f(x) == as_f(y))) break;
        case FB_X_NE_F: FB_BIN((uint64_t)(as_f(x) != as_f(y))) break;
        case FB_X_AND: {  // Kleene: FALSE wins over NULL
          unsigned nv = 0;
          FB_ROWS(const bool va = (accv >> k) & 1u, vb = (bv >> k) & 1u;
                  const bool fa = va && acc[k] == 0, fb = vb && b[k] == 0; const bool isf = fa || fb;
                  if (isf || (va && vb)) nv |= 1u << k; acc[k] = (uint64_t)(!isf && va && vb);)
          accv = nv;
          break;
        }
        case FB_X_OR: {  // Kleene: TRUE wins over NULL
          unsigned nv = 0;
          FB_ROWS(const bool va = (accv >> k) & 1u, vb = (bv >> k) & 1u;
                  const bool ta = va && acc[k] != 0, tb = vb && b[k] != 0; const bool ist = ta || tb;
                  if (ist || (va && vb)) nv |= 1u << k; acc[k] = (uint64_t)ist;)
          accv = nv;
          break;
        }
        case FB_X_COALESCE: FB_ROWS(if (!((accv >> k) & 1u)) acc[k] = b[k];) accv |= bv; break;
        case FB_X_RCOALESCE: FB_ROWS(if ((bv >> k) & 1u) acc[k] = b[k];) accv |= bv; break;
        case FB_X_LOOKUP:
          lookup((const uint64_t*)P.col_ptr[in.b], P.col_valid[in.b], (uint64_t)in.imm, acc, accv);
          break;
        case FB_X_SEL: {  // acc <- temp[flags >> FB_XF_COND_SHIFT] is TRUE ? acc : B
          const int cr = in.flags >> FB_XF_COND_SHIFT;
          const uint64_t* c = tmp_v + (size_t)cr * kExprTile;
          const unsigned cm = tmp_m[cr * kExprThreads + tid];
          unsigned t = 0;
          FB_ROWS(if (((cm >> k) & 1u) && c[k * kExprThreads + tid] != 0) t |= 1u << k; else acc[k] = b[k];)
          accv = (accv & t) | (bv & ~t);
          break;
        }
        case FB_X_MOD_I: FB_CHK(mod_i(acc[k], b[k], acc[k])) break;
        case FB_X_RMOD_I: FB_CHK(mod_i(b[k], acc[k], acc[k])) break;
        case FB_X_MOD_F: FB_CHK(mod_f(acc[k], b[k], acc[k])) break;
        case FB_X_RMOD_F: FB_CHK(mod_f(b[k], acc[k], acc[k])) break;
        case FB_X_ABS_I: FB_UN((int64_t)x < 0 ? 0 - x : x) break;
        case FB_X_ABS_F: FB_UN(x & 0x7FFFFFFFFFFFFFFFull) break;
        case FB_X_FLOOR_F: FB_UN(f_bits(floor(as_f(x)))) break;
        case FB_X_CEIL_F: FB_UN(f_bits(ceil(as_f(x)))) break;
        case FB_X_ROUND_F: FB_UN(f_bits(round_f(as_f(x), (int)in.imm))) break;
        case FB_X_ROUND_I: FB_UN(round_i(x, (int)in.imm)) break;
        case FB_X_SQRT: FB_FUN(sqrt(x)) break;
        case FB_X_EXP: FB_FUN(fn_exp(x)) break;
        case FB_X_LN: FB_FUN(fn_ln(x)) break;
        case FB_X_LOG10: FB_FUN(fn_log10(x)) break;
        case FB_X_POW: FB_FBIN(fn_pow(x, y)) break;
        case FB_X_RPOW: FB_FBIN(fn_pow(y, x)) break;
        case FB_X_GREATEST_I:
          FB_ROWS(if (((bv >> k) & 1u) && (!((accv >> k) & 1u) || (int64_t)b[k] > (int64_t)acc[k])) acc[k] = b[k];)
          accv |= bv;
          break;
        case FB_X_LEAST_I:
          FB_ROWS(if (((bv >> k) & 1u) && (!((accv >> k) & 1u) || (int64_t)b[k] < (int64_t)acc[k])) acc[k] = b[k];)
          accv |= bv;
          break;
        case FB_X_GREATEST_F:
          FB_ROWS(if (((bv >> k) & 1u) && (!((accv >> k) & 1u) || total_key(b[k]) > total_key(acc[k]))) acc[k] = b[k];)
          accv |= bv;
          break;
        case FB_X_LEAST_F:
          FB_ROWS(if (((bv >> k) & 1u) && (!((accv >> k) & 1u) || total_key(b[k]) < total_key(acc[k]))) acc[k] = b[k];)
          accv |= bv;
          break;
        case FB_X_MULSAT_I: FB_BIN(fn_mulsat(x, y)) break;
        case FB_X_FLOORDIV_I: FB_BIN(fn_floordiv(x, y)) break;
        case FB_X_TS_PART: FB_UN(fn_ts_part(x, (int)in.imm)) break;
        case FB_X_TS_TRUNC: FB_UN(fn_ts_trunc(x, (int)in.imm)) break;
        case FB_X_TS_INDEX: FB_UN(fn_ts_index(x, (int)in.imm)) break;
        case FB_X_TS_ADDMON: FB_BIN(fn_ts_addmon(x, y, in.flags >> FB_XF_UNIT_SHIFT)) break;
        default: break;
      }
#undef FB_FBIN
#undef FB_FUN
#undef FB_CHK
#undef FB_BIN
#undef FB_UN
#undef FB_ROWS
    }
  }
}

__global__ void __launch_bounds__(kExprThreads, 3)
fb_eval_expr_kernel(const __grid_constant__ ExprProgram P, int64_t nrows) {
  extern __shared__ __align__(16) uint64_t s_expr[];
  uint64_t* tmp_v = s_expr;                                              // [FB_EXPR_NREGS][kExprTile]
  uint8_t* tmp_m = (uint8_t*)(tmp_v + (size_t)FB_EXPR_NREGS * kExprTile);  // [FB_EXPR_NREGS][kExprThreads] bits
  const int tid = threadIdx.x;
  const int64_t ntiles = (nrows + kExprTile - 1) / kExprTile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * kExprTile;
    if (nrows - row0 >= kExprTile) run_tile<true>(P, row0, kExprTile, tid, tmp_v, tmp_m);
    else run_tile<false>(P, row0, (int)(nrows - row0), tid, tmp_v, tmp_m);
  }
}

constexpr size_t kExprSmem = (size_t)FB_EXPR_NREGS * kExprTile * 8 + (size_t)FB_EXPR_NREGS * kExprThreads;

}  // namespace

extern "C" int fb_eval_expr(int dev, void* stream, int64_t nrows, int ncols, const void* const* col_ptrs,
                            const int32_t* col_types, const uint8_t* const* col_valid, int nins,
                            const fb_expr_ins* program, int nouts, const int32_t* out_types,
                            void* const* out_ptrs, uint8_t* const* out_valid) {
  FB_CHECK(nrows >= 0, "nrows < 0");
  FB_CHECK(ncols >= 0 && ncols <= FB_EXPR_MAX_COLS, "ncols=%d out of range [0,%d]", ncols, FB_EXPR_MAX_COLS);
  FB_CHECK(nins >= 1 && nins <= FB_EXPR_MAX_INS, "nins=%d out of range [1,%d]", nins, FB_EXPR_MAX_INS);
  FB_CHECK(nouts >= 1 && nouts <= FB_EXPR_MAX_OUTS, "nouts=%d out of range [1,%d]", nouts, FB_EXPR_MAX_OUTS);
  FB_CHECK(program != nullptr && out_types != nullptr && out_ptrs != nullptr, "NULL argument");
  ExprProgram P;
  memset(&P, 0, sizeof(P));
  for (int c = 0; c < ncols; ++c) {
    FB_CHECK(col_types[c] >= FB_T_I8 && col_types[c] <= FB_T_F16, "column %d has unknown type %d", c, col_types[c]);
    FB_CHECK(nrows == 0 || col_ptrs[c] != nullptr, "column %d pointer is NULL", c);
    P.col_ptr[c] = col_ptrs[c];
    P.col_type[c] = col_types[c];
    P.col_valid[c] = col_valid ? col_valid[c] : nullptr;
  }
  for (int o = 0; o < nouts; ++o) {
    FB_CHECK(out_types[o] >= FB_T_I8 && out_types[o] <= FB_T_F16, "output %d: unknown type", o);
    FB_CHECK(nrows == 0 || out_ptrs[o] != nullptr, "output %d pointer is NULL", o);
    P.out_type[o] = out_types[o];
    P.out_ptr[o] = out_ptrs[o];
    P.out_valid[o] = out_valid ? out_valid[o] : nullptr;
  }
  for (int i = 0; i < nins; ++i) {
    const fb_expr_ins& in = program[i];
    FB_CHECK(in.op >= FB_X_MOV && in.op <= FB_X_TS_ADDMON, "instruction %d: unknown op %d", i, in.op);
    const bool unary_fn = (in.op >= FB_X_ABS_I && in.op <= FB_X_LOG10) ||  // scalar functions of acc alone
                          (in.op >= FB_X_TS_PART && in.op <= FB_X_TS_INDEX);
    if (unary_fn) FB_CHECK(in.kind == FB_XK_NONE, "instruction %d: op %d takes no operand", i, in.op);
    if (in.op == FB_X_MULSAT_I || in.op == FB_X_FLOORDIV_I)
      FB_CHECK(in.kind == FB_XK_IMM && in.imm >= 1, "instruction %d: op %d takes an immediate >= 1", i, in.op);
    if (in.op >= FB_X_TS_PART && in.op <= FB_X_TS_INDEX) {
      const int64_t nsel = in.op == FB_X_TS_PART ? (int64_t)FB_TF_COUNT : (int64_t)FB_TP_COUNT;
      FB_CHECK(in.imm >= 0 && (in.imm & 0xFF) < nsel && (in.imm >> 8) < FB_TU_COUNT,
               "instruction %d: op %d: field / part %lld or unit %lld out of range", i, in.op,
               (long long)(in.imm & 0xFF), (long long)(in.imm >> 8));
    }
    if (in.op == FB_X_TS_ADDMON)
      FB_CHECK(in.flags >= 0 && (in.flags & 0xFF) == 0 && (in.flags >> FB_XF_UNIT_SHIFT) < FB_TU_COUNT,
               "instruction %d: FB_X_TS_ADDMON flags %#x: the unit in flags >> 8 is out of range", i, in.flags);
    else if (in.op == FB_X_SEL)
      FB_CHECK(in.flags >= 0 && (in.flags >> FB_XF_COND_SHIFT) < FB_EXPR_NREGS,
               "instruction %d: FB_X_SEL condition temporary %d out of range", i, in.flags >> FB_XF_COND_SHIFT);
    else if (in.op > FB_X_LOOKUP)
      FB_CHECK((in.flags & ~FB_XF_B_I2F) == 0, "instruction %d: unknown flags %#x", i, in.flags);
    if (in.op == FB_X_ROUND_F)
      FB_CHECK(in.imm >= -FB_EXPR_ROUND_MAX_DIGITS && in.imm <= FB_EXPR_ROUND_MAX_DIGITS,
               "instruction %d: FB_X_ROUND_F digits %lld out of range", i, (long long)in.imm);
    if (in.op == FB_X_ROUND_I)
      FB_CHECK(in.imm >= -FB_EXPR_ROUND_MAX_DIGITS && in.imm <= -1, "instruction %d: FB_X_ROUND_I digits %lld out of range",
               i, (long long)in.imm);
    if (in.op == FB_X_LOOKUP) {
      FB_CHECK(in.kind == FB_XK_COL, "instruction %d: FB_X_LOOKUP reads a column operand", i);
      FB_CHECK(in.b >= 0 && in.b < ncols, "instruction %d: column %d out of range", i, in.b);
      FB_CHECK(in.imm >= 0, "instruction %d: FB_X_LOOKUP table of %lld entries", i, (long long)in.imm);
      FB_CHECK(col_types[in.b] == FB_T_I64 || col_types[in.b] == FB_T_F64,
               "instruction %d: FB_X_LOOKUP reads a table of 8-byte values, not type %d", i, col_types[in.b]);
    }
    FB_CHECK(in.kind >= FB_XK_NONE && in.kind <= FB_XK_NULL, "instruction %d: unknown operand kind %d", i, in.kind);
    if (in.op == FB_X_ST) {
      FB_CHECK(in.b >= 0 && in.b < FB_EXPR_NREGS, "instruction %d: temporary %d out of range", i, in.b);
      FB_CHECK(in.kind == FB_XK_NONE, "instruction %d: FB_X_ST takes no operand", i);
    } else if (in.op == FB_X_OUT) {
      FB_CHECK(in.b >= 0 && in.b < nouts, "instruction %d: output %d out of range", i, in.b);
      FB_CHECK(in.kind == FB_XK_NONE, "instruction %d: FB_X_OUT takes no operand", i);
    } else if (in.kind == FB_XK_REG) {
      FB_CHECK(in.b >= 0 && in.b < FB_EXPR_NREGS, "instruction %d: temporary %d out of range", i, in.b);
    } else if (in.kind == FB_XK_COL) {
      FB_CHECK(in.b >= 0 && in.b < ncols, "instruction %d: column %d out of range", i, in.b);
    }
    const bool binary = in.op == FB_X_MOV || (in.op >= FB_X_ADD_I && !unary_fn);
    FB_CHECK(!binary || in.kind != FB_XK_NONE, "instruction %d: op %d needs an operand", i, in.op);
    P.ins[i] = in;
  }
  P.nins = nins;
  if (nrows == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  static std::mutex mu;
  static uint64_t optin_done = 0;
  {
    std::lock_guard<std::mutex> lock(mu);
    if (!(dev >= 0 && dev < 64 && ((optin_done >> dev) & 1))) {
      FB_CUDA(cudaFuncSetAttribute(fb_eval_expr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)kExprSmem));
      if (dev >= 0 && dev < 64) optin_done |= 1ull << dev;
    }
  }
  const int64_t ntiles = (nrows + kExprTile - 1) / kExprTile;
  int64_t grid = (int64_t)fb_sm_count(dev) * 3;  // 65 KB of temporaries per CTA: 3 CTAs per SM
  if (grid > ntiles) grid = ntiles;
  fb_eval_expr_kernel<<<(unsigned)grid, kExprThreads, kExprSmem, (cudaStream_t)stream>>>(P, nrows);
  FB_CUDA(cudaGetLastError());
  return 0;
}
