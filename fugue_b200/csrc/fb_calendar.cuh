// Proleptic Gregorian calendar on int64, shared by the expression evaluator (K8: ADD_MONTHS, DATE_TRUNC) and the
// string parser (K13: dates and timestamps), on the device and on the host.  Sums and products are taken on uint64
// (they wrap, never overflow a signed type); every division is by a positive compile-time constant and floors, so
// no instruction can trap.
#pragma once
#include "fb_common.cuh"

FB_HD int64_t wadd(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
FB_HD int64_t wsub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
FB_HD int64_t wmul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
template <int64_t C>
FB_HD int64_t fdiv(int64_t x) {  // floor(x / C)
  const int64_t q = x / C;
  return q - (int64_t)(x % C < 0);
}

FB_HD bool is_leap(int64_t y) { return (y & 3) == 0 && (y % 100 != 0 || y % 400 == 0); }

// year, month (1-12), day (1-31) -> days since 1970-01-01: 400-year eras of 146 097 days, years that start on March 1
FB_HD int64_t days_from_civil(int64_t y, int m, int d) {
  y = wsub(y, (int64_t)(m <= 2));
  const int64_t era = fdiv<400ll>(y);
  const int yoe = (int)wsub(y, wmul(era, 400ll));                                // [0, 399]
  const int doy_m = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
  const int doe = yoe * 365 + yoe / 4 - yoe / 100 + doy_m;
  return wsub(wadd(wmul(era, 146097ll), (int64_t)doe), 719468ll);
}
