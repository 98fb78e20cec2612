// K14 format routines: one 8-byte value -> its UTF-8 text, the text the host frames write for a cast to string
// (include/fugue_b200.h, DESIGN.md section 7n).  FB_HD: the kernel and the host export run these same functions.
//
// Every routine writes through a sink: FbCount only counts the bytes, FbStore also stores them, so the measure and
// the write call of fb_value_format cannot disagree on a length.
//
// Floats: the shortest digits that read back to the same float64 (Ryu, Adams 2018), laid out as CPython's repr.
// Dates and timestamps: Arrow's cast to string and strftime("%Y-%m-%d %H:%M:%S"), including what they write where
// their calendar arithmetic wraps (32-bit days, 16-bit years).
#pragma once
#include "fb_calendar.cuh"

static const uint64_t fb_ryu_host[][2] = {
#include "fb_ryu.inc"
};
#ifdef __CUDACC__
static __device__ const uint64_t fb_ryu_dev[][2] = {
#include "fb_ryu.inc"
};
#endif
#define FB_RYU_INV_ROWS 342
#define FB_RYU_POW_ROWS 326
static_assert(sizeof(fb_ryu_host) / sizeof(fb_ryu_host[0]) == FB_RYU_INV_ROWS + FB_RYU_POW_ROWS, "fb_ryu.inc rows");

// Arrow prints a date32 outside these days (years -32767 .. 32767) as "<value out of range: n>"
#define FB_FMT_DAY_MIN (-12687428ll)
#define FB_FMT_DAY_MAX 11248737ll

struct FbCount {
  int64_t n = 0;
  FB_HD void put(uint8_t) { ++n; }
  FB_HD void digits(uint64_t, int nd) { n += nd; }
};

struct FbStore {
  uint8_t* p;
  int64_t n = 0;
  FB_HD void put(uint8_t c) { p[n++] = c; }
  FB_HD void digits(uint64_t v, int nd) {  // the low nd decimal digits of v, most significant first
    for (int k = nd - 1; k >= 0; --k) {
      p[n + k] = (uint8_t)('0' + v % 10);
      v /= 10;
    }
    n += nd;
  }
};

FB_HD int fb_ndigits(uint64_t v) {
  int nd = 1;
  for (; v >= 10; v /= 10) ++nd;
  return nd;
}

template <class S>
FB_HD void fb_put_uint(S& s, uint64_t v, int min_digits = 1) {
  const int nd = fb_ndigits(v);
  s.digits(v, nd < min_digits ? min_digits : nd);
}

template <class S>
FB_HD void fb_put_int(S& s, int64_t v, int min_digits = 1) {
  if (v < 0) s.put('-');
  fb_put_uint(s, v < 0 ? 0 - (uint64_t)v : (uint64_t)v, min_digits);
}

template <class S>
FB_HD void fb_put_word(S& s, const char* w) {
  for (; *w != 0; ++w) s.put((uint8_t)*w);
}

// ---- float64: Ryu's shortest decimal w * 10^e10 inside the rounding interval, nearest to the value
FB_HD void fb_ryu_row(int r, uint64_t& hi, uint64_t& lo) {
#ifdef __CUDA_ARCH__
  hi = __ldg((const unsigned long long*)&fb_ryu_dev[r][0]);
  lo = __ldg((const unsigned long long*)&fb_ryu_dev[r][1]);
#else
  hi = fb_ryu_host[r][0];
  lo = fb_ryu_host[r][1];
#endif
}

FB_HD uint32_t fb_pow5bits(int32_t e) { return (uint32_t)(((uint32_t)e * 1217359u) >> 19) + 1; }  // bitlen(5^e)
FB_HD uint32_t fb_log10_pow2(int32_t e) { return ((uint32_t)e * 78913u) >> 18; }
FB_HD uint32_t fb_log10_pow5(int32_t e) { return ((uint32_t)e * 732923u) >> 20; }

FB_HD bool fb_multiple_of_pow5(uint64_t v, uint32_t p) {
  uint32_t k = 0;
  for (; v != 0 && v % 5 == 0; v /= 5) ++k;
  return k >= p;
}

// (m * {hi, lo}) >> j of a 125-bit multiplier, 64 < j < 128
FB_HD uint64_t fb_ryu_mulshift(uint64_t m, uint64_t hi, uint64_t lo, int32_t j) {
  const uint64_t b0 = fb_mulhi64(m, lo);
  const uint64_t s_lo = m * hi + b0;
  const uint64_t s_hi = fb_mulhi64(m, hi) + (s_lo < b0);
  const int sh = j - 64;
  return (s_lo >> sh) | (s_hi << (64 - sh));
}

// finite, non-zero float64 bits (no sign) -> (digits, e10)
FB_HD void fb_ryu_d2d(uint64_t mant, uint32_t expo, uint64_t& digits, int32_t& e10) {
  int32_t e2;
  uint64_t m2;
  if (expo == 0) {
    e2 = 1 - 1023 - 52 - 2;
    m2 = mant;
  } else {
    e2 = (int32_t)expo - 1023 - 52 - 2;
    m2 = (1ull << 52) | mant;
  }
  const bool accept = (m2 & 1) == 0;
  const uint64_t mv = 4 * m2;
  const uint32_t mm_shift = mant != 0 || expo <= 1;
  uint64_t vr, vp, vm, hi, lo;
  bool vm_zeros = false, vr_zeros = false;
  if (e2 >= 0) {
    const uint32_t q = fb_log10_pow2(e2) - (e2 > 3);
    e10 = (int32_t)q;
    const int32_t k = 125 + (int32_t)fb_pow5bits((int32_t)q) - 1;
    const int32_t i = -e2 + (int32_t)q + k;
    fb_ryu_row((int)q, hi, lo);
    vr = fb_ryu_mulshift(4 * m2, hi, lo, i);
    vp = fb_ryu_mulshift(4 * m2 + 2, hi, lo, i);
    vm = fb_ryu_mulshift(4 * m2 - 1 - mm_shift, hi, lo, i);
    if (q <= 21) {
      if (mv % 5 == 0) vr_zeros = fb_multiple_of_pow5(mv, q);
      else if (accept) vm_zeros = fb_multiple_of_pow5(mv - 1 - mm_shift, q);
      else vp -= fb_multiple_of_pow5(mv + 2, q);
    }
  } else {
    const uint32_t q = fb_log10_pow5(-e2) - (-e2 > 1);
    e10 = (int32_t)q + e2;
    const int32_t i = -e2 - (int32_t)q;
    const int32_t k = (int32_t)fb_pow5bits(i) - 125;
    const int32_t j = (int32_t)q - k;
    fb_ryu_row(FB_RYU_INV_ROWS + i, hi, lo);
    vr = fb_ryu_mulshift(4 * m2, hi, lo, j);
    vp = fb_ryu_mulshift(4 * m2 + 2, hi, lo, j);
    vm = fb_ryu_mulshift(4 * m2 - 1 - mm_shift, hi, lo, j);
    if (q <= 1) {
      vr_zeros = true;
      if (accept) vm_zeros = mm_shift == 1;
      else --vp;
    } else if (q < 63) {
      vr_zeros = (mv & ((1ull << q) - 1)) == 0;
    }
  }
  int32_t removed = 0;
  uint32_t last = 0;
  while (vp / 10 > vm / 10) {
    vm_zeros &= vm % 10 == 0;
    vr_zeros &= last == 0;
    last = (uint32_t)(vr % 10);
    vr /= 10;
    vp /= 10;
    vm /= 10;
    ++removed;
  }
  if (vm_zeros) {
    while (vm % 10 == 0) {
      vr_zeros &= last == 0;
      last = (uint32_t)(vr % 10);
      vr /= 10;
      vp /= 10;
      vm /= 10;
      ++removed;
    }
  }
  if (vr_zeros && last == 5 && vr % 2 == 0) last = 4;  // exactly halfway: round to even
  digits = vr + ((vr == vm && (!accept || !vm_zeros)) || last >= 5);
  e10 += removed;
}

// CPython's repr(float): fixed notation when the decimal exponent x of the first digit is in [-4, 16), else
// d[.ddd]e(+|-)XX
template <class S>
FB_HD void fb_put_f64(S& s, uint64_t bits) {
  const bool neg = bits >> 63;
  const uint32_t expo = (uint32_t)(bits >> 52) & 0x7FF;
  const uint64_t mant = bits & ((1ull << 52) - 1);
  if (expo == 0x7FF) {
    if (mant != 0) return fb_put_word(s, "nan");
    return fb_put_word(s, neg ? "-inf" : "inf");
  }
  if (neg) s.put('-');
  if (expo == 0 && mant == 0) return fb_put_word(s, "0.0");
  uint64_t d;
  int32_t e10;
  fb_ryu_d2d(mant, expo, d, e10);
  const int nd = fb_ndigits(d);
  const int x = e10 + nd - 1;
  if (x >= -4 && x < 16) {
    if (x < 0) {
      fb_put_word(s, "0.");
      for (int k = 0; k < -x - 1; ++k) s.put('0');
      s.digits(d, nd);
    } else if (nd <= x + 1) {  // an integer: its digits, the zeros to the decimal point, ".0"
      s.digits(d, nd);
      for (int k = nd; k <= x; ++k) s.put('0');
      fb_put_word(s, ".0");
    } else {
      uint64_t p = 1;
      for (int k = 0; k < nd - x - 1; ++k) p *= 10;
      s.digits(d / p, x + 1);
      s.put('.');
      s.digits(d % p, nd - x - 1);
    }
    return;
  }
  uint64_t p = 1;
  for (int k = 1; k < nd; ++k) p *= 10;
  s.digits(d / p, 1);
  if (nd > 1) {
    s.put('.');
    s.digits(d % p, nd - 1);
  }
  s.put('e');
  s.put(x < 0 ? '-' : '+');
  fb_put_uint(s, (uint64_t)(x < 0 ? -x : x), 2);
}

// ---- dates and timestamps: the civil date of day z as the vendored date library computes it, in 32-bit arithmetic
// with the year kept in 16 bits (both wrap, as in Arrow)
FB_HD void fb_civil_from_days32(int32_t z0, int& y, int& m, int& d) {
  const int32_t z = (int32_t)((uint32_t)z0 + 719468u);
  const int32_t era = (z >= 0 ? z : (int32_t)((uint32_t)z - 146096u)) / 146097;
  const uint32_t doe = (uint32_t)z - (uint32_t)era * 146097u;
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const int32_t yy = (int32_t)(yoe + (uint32_t)era * 400u);
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint32_t mp = (5 * doy + 2) / 153;
  d = (int)(doy - (153 * mp + 2) / 5 + 1);
  m = (int)(mp < 10 ? mp + 3 : mp - 9);
  y = (int16_t)(uint16_t)(uint32_t)(yy + (m <= 2));
}

template <class S>
FB_HD void fb_put_ymd(S& s, int32_t days) {
  int y, m, d;
  fb_civil_from_days32(days, y, m, d);
  fb_put_int(s, y, 4);
  s.put('-');
  fb_put_uint(s, (uint64_t)m, 2);
  s.put('-');
  fb_put_uint(s, (uint64_t)d, 2);
}

// days: the floor day, checked against the range; text_day: the day written (a date64 truncates toward 0, as Arrow)
template <class S>
FB_HD void fb_put_date(S& s, int64_t raw, int64_t days, int64_t text_day) {
  if (days < FB_FMT_DAY_MIN || days > FB_FMT_DAY_MAX) {
    fb_put_word(s, "<value out of range: ");
    fb_put_int(s, raw);
    s.put('>');
    return;
  }
  fb_put_ymd(s, (int32_t)text_day);
}

// YYYY-MM-DD HH:MM:SS[.fraction]: the day is floor(t / day) cut to 32 bits, the time of day t minus that day's start
// (its hours run past 23 where the day wrapped, and carry the sign when the time of day is negative)
template <class S>
FB_HD void fb_put_timestamp(S& s, int64_t t, int unit, bool frac) {
  const int64_t per = unit == FB_TU_S ? 1 : unit == FB_TU_MS ? 1000 : unit == FB_TU_US ? 1000000 : 1000000000;
  const int64_t pd = 86400 * per;
  int32_t day = (int32_t)(uint32_t)(uint64_t)(t / pd);
  if (wmul(day, pd) > t) day = (int32_t)((uint32_t)day - 1u);
  const int64_t tod = wsub(t, wmul(day, pd));
  const uint64_t a = tod < 0 ? 0 - (uint64_t)tod : (uint64_t)tod;
  const uint64_t h = a / (uint64_t)(3600 * per);
  uint64_t r = a - h * (uint64_t)(3600 * per);
  const uint64_t mi = r / (uint64_t)(60 * per);
  r -= mi * (uint64_t)(60 * per);
  const uint64_t sec = r / (uint64_t)per;
  fb_put_ymd(s, day);
  s.put(' ');
  if (tod < 0) s.put('-');
  fb_put_uint(s, h, 2);
  s.put(':');
  fb_put_uint(s, mi, 2);
  s.put(':');
  fb_put_uint(s, sec, 2);
  if (frac) {
    s.put('.');
    fb_put_uint(s, r - sec * (uint64_t)per, unit == FB_TU_MS ? 3 : unit == FB_TU_US ? 6 : 9);
  }
}

// one value of a kind (FB_FMT_*) -> its text
template <class S>
FB_HD void fb_format_value(S& s, uint64_t v, int kind) {
  switch (kind) {
    case FB_FMT_I64: return fb_put_int(s, (int64_t)v);
    case FB_FMT_U64: return fb_put_uint(s, v);
    case FB_FMT_BOOL: return fb_put_word(s, v != 0 ? "true" : "false");
    case FB_FMT_F64: return fb_put_f64(s, v);
    case FB_FMT_DATE32: return fb_put_date(s, (int64_t)v, (int64_t)v, (int64_t)v);
    case FB_FMT_DATE64: return fb_put_date(s, (int64_t)v, fdiv<86400000ll>((int64_t)v), (int64_t)v / 86400000);
    default: return fb_put_timestamp(s, (int64_t)v, kind & 7, (kind & FB_FMT_TS_FRAC) != 0);
  }
}
