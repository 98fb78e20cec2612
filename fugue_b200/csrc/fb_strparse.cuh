// K13 parse routines: one string entry -> one typed value, bit for bit what Arrow's cast(safe=False) of the string
// gives (include/fugue_b200.h, DESIGN.md section 7l).  FB_HD: the kernel and the host export run these same
// functions.
//
// Floats: Clinger's exact fast path when the significand and the power of ten are both exact in the target, else
// the Eisel-Lemire algorithm over 128-bit truncated powers of five (Lemire 2021; Mushtak & Lemire 2023 show that
// it needs no fallback while the significand fits in 64 bits, i.e. up to 19 significant digits).  A longer
// significand is truncated to 19 digits w; w and w + 1 bracket the value, and when both round to the same float
// that is the answer, else the entry is FB_PARSE_UNDECIDED.
#pragma once
#include "fb_calendar.cuh"

static const uint64_t fb_pow5_host[][2] = {
#include "fb_pow5.inc"
};
#ifdef __CUDACC__
static __device__ const uint64_t fb_pow5_dev[][2] = {
#include "fb_pow5.inc"
};
#endif
#define FB_POW5_QMIN (-342)
#define FB_POW5_QMAX 308
static_assert(sizeof(fb_pow5_host) / sizeof(fb_pow5_host[0]) == FB_POW5_QMAX - FB_POW5_QMIN + 1, "fb_pow5.inc rows");

FB_HD void fb_pow5(int q, uint64_t& hi, uint64_t& lo) {
#ifdef __CUDA_ARCH__
  hi = __ldg((const unsigned long long*)&fb_pow5_dev[q - FB_POW5_QMIN][0]);
  lo = __ldg((const unsigned long long*)&fb_pow5_dev[q - FB_POW5_QMIN][1]);
#else
  hi = fb_pow5_host[q - FB_POW5_QMIN][0];
  lo = fb_pow5_host[q - FB_POW5_QMIN][1];
#endif
}

FB_HD uint64_t fb_f64_bits(double d) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t b;
  memcpy(&b, &d, 8);
  return b;
#endif
}
FB_HD uint32_t fb_f32_bits(float f) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, 4);
  return b;
#endif
}
FB_HD float fb_f32_from(uint32_t b) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}

FB_HD bool fb_is_digit(uint8_t c) { return (uint8_t)(c - '0') < 10; }
FB_HD uint8_t fb_lower(uint8_t c) { return (uint8_t)(c - 'A') < 26 ? (uint8_t)(c | 0x20) : c; }

// s[0, n) equals the lower-case ASCII word w, ignoring case
FB_HD bool fb_word_ci(const uint8_t* s, int64_t n, const char* w) {
  int64_t i = 0;
  for (; w[i] != 0; ++i)
    if (i >= n || fb_lower(s[i]) != (uint8_t)w[i]) return false;
  return i == n;
}

// ---- integers: decimal with an optional '-', or 0x / 0X hex of at most 2 * bytes digits read as two's complement
FB_HD uint8_t fb_parse_int(const uint8_t* s, int64_t n, int bytes, bool is_signed, uint64_t& out) {
  const int bits = bytes * 8;
  if (n >= 2 && s[0] == '0' && (s[1] | 0x20) == 'x') {
    const int64_t nd = n - 2;
    if (nd < 1 || nd > 2 * bytes) return FB_PARSE_INVALID;
    uint64_t v = 0;
    for (int64_t i = 2; i < n; ++i) {
      const uint8_t c = s[i], l = fb_lower(c);
      int d;
      if (fb_is_digit(c)) d = c - '0';
      else if (l >= 'a' && l <= 'f') d = l - 'a' + 10;
      else return FB_PARSE_INVALID;
      v = v << 4 | (uint64_t)d;
    }
    if (is_signed && bits < 64 && ((v >> (bits - 1)) & 1)) v |= ~0ull << bits;  // sign-extend
    out = v;
    return FB_PARSE_OK;
  }
  const bool neg = n > 0 && s[0] == '-';
  if (neg && !is_signed) return FB_PARSE_INVALID;
  int64_t i = neg ? 1 : 0;
  if (i >= n) return FB_PARSE_INVALID;
  uint64_t v = 0;
  for (; i < n; ++i) {
    if (!fb_is_digit(s[i])) return FB_PARSE_INVALID;
    const uint64_t d = s[i] - '0';
    if (v > (~0ull - d) / 10) return FB_PARSE_INVALID;  // beyond uint64
    v = v * 10 + d;
  }
  const uint64_t lim = is_signed ? (1ull << (bits - 1)) - (neg ? 0 : 1) : (bits == 64 ? ~0ull : (1ull << bits) - 1);
  if (v > lim) return FB_PARSE_INVALID;
  out = neg ? 0 - v : v;
  return FB_PARSE_OK;
}

// ---- booleans: true / false in any case, 1, 0
FB_HD uint8_t fb_parse_bool(const uint8_t* s, int64_t n, uint64_t& out) {
  if (n == 1 && (s[0] == '0' || s[0] == '1')) {
    out = s[0] - '0';
    return FB_PARSE_OK;
  }
  if (fb_word_ci(s, n, "true")) { out = 1; return FB_PARSE_OK; }
  if (fb_word_ci(s, n, "false")) { out = 0; return FB_PARSE_OK; }
  return FB_PARSE_INVALID;
}

// ---- floats
struct FbFloatFormat {
  int mbits;          // explicit mantissa bits
  int min_exp;        // -bias
  int inf_power;      // biased exponent of infinity
  int q_min, q_max;   // below: zero; above: infinity (for any 64-bit significand)
  int even_lo, even_hi;  // the q for which a product can be exactly halfway between two floats
};
#define FB_F64_FORMAT FbFloatFormat{52, -1023, 0x7FF, -342, 308, -4, 23}
#define FB_F32_FORMAT FbFloatFormat{23, -127, 0xFF, -65, 38, -17, 10}

// Eisel-Lemire: the IEEE bits (without sign) of w * 10^q correctly rounded, w != 0
FB_HD uint64_t fb_eisel_lemire(uint64_t w, int64_t q, const FbFloatFormat F) {
  if (q < F.q_min) return 0;
  if (q > F.q_max) return (uint64_t)F.inf_power << F.mbits;
#ifdef __CUDA_ARCH__
  const int lz = __clzll((long long)w);
#else
  const int lz = __builtin_clzll(w);
#endif
  w <<= lz;
  uint64_t p_hi, p_lo;
  fb_pow5((int)q, p_hi, p_lo);
  uint64_t hi = fb_mulhi64(w, p_hi), lo = w * p_hi;
  const uint64_t mask = ~0ull >> (F.mbits + 3);
  if ((hi & mask) == mask) {  // the low bits of the top word might still carry: add the second word's product
    const uint64_t h2 = fb_mulhi64(w, p_lo);
    lo += h2;
    if (h2 > lo) ++hi;
  }
  const int upper = (int)(hi >> 63);
  const int shift = upper + 64 - F.mbits - 3;
  uint64_t m = hi >> shift;
  // floor(q * log2(10)) + 63, exact for |q| <= 1500
  int p2 = (int)((((152170 + 65536) * (int64_t)q) >> 16) + 63) + upper - lz - F.min_exp;
  if (p2 <= 0) {  // subnormal
    if (-p2 + 1 >= 64) return 0;
    m >>= -p2 + 1;
    m += m & 1;
    m >>= 1;
    return m < (1ull << F.mbits) ? m : (1ull << F.mbits);  // rounding up to the smallest normal gives exponent 1
  }
  if (lo <= 1 && q >= F.even_lo && q <= F.even_hi && (m & 3) == 1 && (m << shift) == hi) m &= ~1ull;  // ties to even
  m += m & 1;
  m >>= 1;
  if (m >= (2ull << F.mbits)) {
    m = 1ull << F.mbits;
    ++p2;
  }
  m &= ~(1ull << F.mbits);
  if (p2 >= F.inf_power) return (uint64_t)F.inf_power << F.mbits;
  return m | (uint64_t)p2 << F.mbits;
}

// w * 10^q correctly rounded to the target (no sign); Clinger's exact path when both factors are exact
FB_HD uint64_t fb_decimal_to_bits(uint64_t w, int64_t q, bool f32) {
  if (w == 0) return 0;
  if (f32) {
    if (w <= (1ull << 24) && q >= -10 && q <= 10) {
      float p = 1.0f;
      for (int i = 0; i < (q < 0 ? -q : q); ++i) p *= 10.0f;
      return fb_f32_bits(q < 0 ? (float)w / p : (float)w * p);
    }
    return fb_eisel_lemire(w, q, FB_F32_FORMAT);
  }
  if (w <= (1ull << 53) && q >= -22 && q <= 22) {
    double p = 1.0;
    for (int i = 0; i < (q < 0 ? -q : q); ++i) p *= 10.0;
    return fb_f64_bits(q < 0 ? (double)w / p : (double)w * p);
  }
  return fb_eisel_lemire(w, q, FB_F64_FORMAT);
}

// out: the value's float64 bits (a float32 target gives its exact widening, which FB_X_LOOKUP reads as float64)
FB_HD uint8_t fb_parse_float(const uint8_t* s, int64_t n, bool f32, uint64_t& out) {
  int64_t i = 0;
  const bool neg = n > 0 && s[0] == '-';
  if (n > 0 && (s[0] == '-' || s[0] == '+')) i = 1;
  const uint64_t sign32 = neg ? 1ull << 31 : 0, sign64 = neg ? 1ull << 63 : 0;
  const uint8_t* r = s + i;
  const int64_t m = n - i;
  if (m >= 3 && (fb_lower(r[0]) == 'i' || fb_lower(r[0]) == 'n')) {
    if (fb_word_ci(r, m, "inf") || fb_word_ci(r, m, "infinity")) {
      out = sign64 | 0x7FF0000000000000ull;
      return FB_PARSE_OK;
    }
    bool nan = fb_word_ci(r, m, "nan");
    if (!nan && m >= 5 && fb_word_ci(r, 3, "nan") && r[3] == '(' && r[m - 1] == ')') {  // nan(n-char-sequence)
      nan = true;
      for (int64_t k = 4; k < m - 1; ++k) {
        const uint8_t c = fb_lower(r[k]);
        if (!(fb_is_digit(c) || (c >= 'a' && c <= 'z') || c == '_')) nan = false;
      }
    }
    if (nan) {
      out = sign64 | 0x7FF8000000000000ull;
      return FB_PARSE_OK;
    }
    return FB_PARSE_INVALID;
  }
  uint64_t w = 0;
  int nd = 0;           // significant digits kept in w (at most 19)
  int64_t dexp = 0;     // the value is (w + a fraction when truncated) * 10^(dexp + exponent)
  bool started = false, truncated = false, any = false;
  for (; i < n && fb_is_digit(s[i]); ++i) {
    const int d = s[i] - '0';
    any = true;
    if (!started && d == 0) continue;
    started = true;
    if (nd < 19) {
      w = w * 10 + d;
      ++nd;
    } else {
      ++dexp;
      truncated |= d != 0;
    }
  }
  if (i < n && s[i] == '.') {
    for (++i; i < n && fb_is_digit(s[i]); ++i) {
      const int d = s[i] - '0';
      any = true;
      if (!started && d == 0) {
        --dexp;
        continue;
      }
      started = true;
      if (nd < 19) {
        w = w * 10 + d;
        ++nd;
        --dexp;
      } else {
        truncated |= d != 0;
      }
    }
  }
  if (!any) return FB_PARSE_INVALID;
  if (i < n && (s[i] | 0x20) == 'e') {
    ++i;
    bool eneg = false;
    if (i < n && (s[i] == '-' || s[i] == '+')) eneg = s[i++] == '-';
    if (i >= n || !fb_is_digit(s[i])) return FB_PARSE_INVALID;
    int64_t e = 0;
    for (; i < n && fb_is_digit(s[i]); ++i)
      if (e < 100000000000ll) e = e * 10 + (s[i] - '0');  // saturates far beyond every finite float
    dexp += eneg ? -e : e;
  }
  if (i != n) return FB_PARSE_INVALID;
  uint64_t b = fb_decimal_to_bits(w, dexp, f32);
  if (truncated && fb_decimal_to_bits(w + 1, dexp, f32) != b) return FB_PARSE_UNDECIDED;
  if (f32) {
    out = fb_f64_bits((double)fb_f32_from((uint32_t)b | (uint32_t)sign32));
  } else {
    out = b | sign64;
  }
  return FB_PARSE_OK;
}

// ---- dates and timestamps
FB_HD int fb_digits(const uint8_t* s, int k) {  // k decimal digits as an int, or -1
  int v = 0;
  for (int i = 0; i < k; ++i) {
    if (!fb_is_digit(s[i])) return -1;
    v = v * 10 + (s[i] - '0');
  }
  return v;
}

// exactly YYYY-MM-DD with a valid calendar day -> days since 1970-01-01
FB_HD bool fb_parse_ymd(const uint8_t* s, int64_t n, int64_t& days) {
  if (n < 10 || s[4] != '-' || s[7] != '-') return false;
  const int y = fb_digits(s, 4), mo = fb_digits(s + 5, 2), d = fb_digits(s + 8, 2);
  if (y < 0 || mo < 1 || mo > 12 || d < 1) return false;
  const int last = mo == 2 ? 28 + (int)is_leap(y) : 30 + ((mo + (mo >> 3)) & 1);
  if (d > last) return false;
  days = days_from_civil(y, mo, d);
  return true;
}

FB_HD bool fb_mul_ok(int64_t a, int64_t b, int64_t& r) {  // r = a * b for b > 0; false on int64 overflow
  if (a > INT64_MAX / b || a < INT64_MIN / b) return false;
  r = a * b;
  return true;
}

// YYYY-MM-DD[(T| )HH[:MM[:SS[.f{1,9}]]]] then, when zoned, a required Z / +-HH / +-HHMM / +-HH:MM after the time
FB_HD uint8_t fb_parse_timestamp(const uint8_t* s, int64_t n, int unit, bool zoned, uint64_t& out) {
  int64_t days;
  if (!fb_parse_ymd(s, n, days)) return FB_PARSE_INVALID;
  int64_t secs = days * 86400, frac = 0;  // frac: in the unit
  int64_t i = 10;
  if (n == 10) {
    if (zoned) return FB_PARSE_INVALID;
  } else {
    if (s[10] != 'T' && s[10] != ' ') return FB_PARSE_INVALID;
    if (n < 13) return FB_PARSE_INVALID;
    const int h = fb_digits(s + 11, 2);
    if (h < 0 || h > 23) return FB_PARSE_INVALID;
    int mi = 0, se = 0;
    i = 13;
    if (i < n && s[i] == ':') {
      if (n < i + 3 || (mi = fb_digits(s + i + 1, 2)) < 0 || mi > 59) return FB_PARSE_INVALID;
      i += 3;
      if (i < n && s[i] == ':') {
        if (n < i + 3 || (se = fb_digits(s + i + 1, 2)) < 0 || se > 59) return FB_PARSE_INVALID;
        i += 3;
        if (i < n && s[i] == '.') {
          const int maxd = unit == FB_TU_S ? 0 : unit == FB_TU_MS ? 3 : unit == FB_TU_US ? 6 : 9;
          int nd = 0;
          for (++i; i < n && fb_is_digit(s[i]); ++i, ++nd) {
            if (nd >= maxd) return FB_PARSE_INVALID;
            frac = frac * 10 + (s[i] - '0');
          }
          if (nd == 0) return FB_PARSE_INVALID;
          for (; nd < maxd; ++nd) frac *= 10;
        }
      }
    }
    secs += h * 3600 + mi * 60 + se;
    if (zoned) {
      if (i >= n) return FB_PARSE_INVALID;
      if (s[i] == 'Z') {
        ++i;
      } else if (s[i] == '+' || s[i] == '-') {
        const int64_t sign = s[i] == '-' ? -1 : 1;
        const int64_t k = n - i - 1;  // 2, 4 or 5 characters
        const int oh = k >= 2 ? fb_digits(s + i + 1, 2) : -1;
        int om = 0;
        if (k == 4) om = fb_digits(s + i + 3, 2);
        else if (k == 5) om = s[i + 3] == ':' ? fb_digits(s + i + 4, 2) : -1;
        else if (k != 2) return FB_PARSE_INVALID;
        if (oh < 0 || oh > 23 || om < 0 || om > 59) return FB_PARSE_INVALID;
        secs -= sign * (oh * 3600 + om * 60);
        i = n;
      } else {
        return FB_PARSE_INVALID;
      }
    }
    if (i != n) return FB_PARSE_INVALID;
  }
  const int64_t per = unit == FB_TU_S ? 1 : unit == FB_TU_MS ? 1000 : unit == FB_TU_US ? 1000000 : 1000000000;
  int64_t v;
  if (!fb_mul_ok(secs, per, v) || v > INT64_MAX - frac) return FB_PARSE_INVALID;
  out = (uint64_t)(v + frac);
  return FB_PARSE_OK;
}

// one entry -> (status, the 8-byte word FB_X_LOOKUP reads)
FB_HD uint8_t fb_parse_entry(const uint8_t* s, int64_t n, int target, uint64_t& out) {
  out = 0;
  if (target >= FB_PARSE_I8 && target <= FB_PARSE_U64)
    return fb_parse_int(s, n, 1 << (target & 3), target <= FB_PARSE_I64, out);
  switch (target) {
    case FB_PARSE_F32: return fb_parse_float(s, n, true, out);
    case FB_PARSE_F64: return fb_parse_float(s, n, false, out);
    case FB_PARSE_BOOL: return fb_parse_bool(s, n, out);
    case FB_PARSE_DATE32:
    case FB_PARSE_DATE64: {
      int64_t days;
      if (n != 10 || !fb_parse_ymd(s, n, days)) return FB_PARSE_INVALID;
      out = (uint64_t)(target == FB_PARSE_DATE64 ? days * 86400000ll : days);
      return FB_PARSE_OK;
    }
    default: break;
  }
  const int unit = target & 7;
  return fb_parse_timestamp(s, n, unit, (target & FB_PARSE_TS_ZONED) != 0, out);
}
