"""What each aggregate function means at run time, written once for the hash group-by (K6) and the window scans (K9).

The two routes reduce differently - K6 accumulates per group, K9 scans per row of a logical partition - but they pick
the same kernel op for a function, feed it the same 8-byte values, and finish its raw state with the same torch
expressions.  Those per-function parts live here; the routes keep only how they plan and launch their reductions.
Which heads exist and their result types are in ``column.AGGREGATES``.
"""
import math
from typing import Any, Dict, Optional, Sequence, Tuple

import pyarrow as pa
import torch

from . import kernels as K
from . import sort as S
from .column import AGGREGATES, EWM_HEADS, result_type
from .table import B200Table, narrow, widen

# (function, values are float64) -> the K6 / K9 op; FIRST / LAST reduce the row numbers of the valid rows
_OPS = {("SUM", False): K.AGG_SUM_I64, ("SUM", True): K.AGG_SUM_F64, ("AVG", True): K.AGG_SUM_F64,
        ("MIN", False): K.AGG_MIN_I64, ("MIN", True): K.AGG_MIN_F64,
        ("MAX", False): K.AGG_MAX_I64, ("MAX", True): K.AGG_MAX_F64,
        ("FIRST", False): K.AGG_MIN_I64, ("LAST", False): K.AGG_MAX_I64}


def check_argument(fn: str, name: str, tp: pa.DataType, is_dictionary: bool) -> None:
    """Reject an argument column ``name`` of arrow type ``tp`` that ``fn`` does not take: the variances and the
    shape statistics and the two-argument functions need integer or float columns, and a string column takes no SUM
    or AVG."""
    if fn in EWM_HEADS or AGGREGATES[fn].family in ("variance", "shape", "bivariate"):
        if is_dictionary or not (pa.types.is_integer(tp) or pa.types.is_floating(tp)):
            raise NotImplementedError(f"{fn} needs integer or float columns; {name} is {tp}")
    elif is_dictionary and fn in ("SUM", "AVG"):
        raise NotImplementedError(f"{fn} on the string column {name}: strings take MIN and MAX")


def f64_values(t: B200Table, name: str, cache: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
    """Column ``name`` of ``t`` widened to contiguous float64 as AVG reads it.  With ``cache``, once per name: K6 ties a
    DEV / DEV2 / CODEV to its column by data pointer, so one call must give every use of a column the same tensor
    (DESIGN §7i)."""
    if cache is None:
        i = t.schema.index_of_key(name)
        return reduce_input("AVG", t.columns[i], t.schema.types[i])[1]
    if name not in cache:
        cache[name] = f64_values(t, name)
    return cache[name]


def reduce_input(fn: str, c: torch.Tensor, tp: pa.DataType) -> Tuple[int, torch.Tensor]:
    """(op, contiguous 8-byte values) that reduce column ``c`` of arrow type ``tp`` for SUM / AVG / MIN / MAX, and
    for FIRST / LAST of the row numbers (int64).  AVG sums float64; the others keep the integer or float class."""
    if fn == "AVG":
        return _OPS[(fn, True)], widen(c, tp).to(torch.float64).contiguous()
    return _OPS[(fn, pa.types.is_floating(tp))], widen(c, tp).contiguous()


def divides_by_count(fn: str) -> bool:
    """Whether ``finish_basic`` needs the count of ``fn`` even where the result is never NULL: AVG divides by it."""
    return fn == "AVG"


def finish_basic(fn: str, value: Optional[torch.Tensor], count: Optional[torch.Tensor],
                 tp: Optional[pa.DataType]) -> Tuple[torch.Tensor, Optional[torch.Tensor], pa.DataType]:
    """(column, validity, type) of SUM / AVG / MIN / MAX / COUNT of an argument of arrow type ``tp`` from the reduced
    ``value`` (float64 or int64, as ``reduce_input`` chose; unused by COUNT) and the non-NULL ``count``.  The result is
    NULL where the count is 0; ``count=None``: never NULL (a keyed aggregate of a column without NULLs)."""
    out = result_type(fn, tp)
    if fn == "COUNT":
        return count.contiguous(), None, out
    valid = None if count is None else (count > 0).to(torch.uint8)
    if fn == "AVG":
        value = value / count.to(torch.float64)
    return narrow(value, out).contiguous(), valid, out


def finish_string(ranks: torch.Tensor, count: torch.Tensor, d: pa.Array, tp: pa.DataType) -> Tuple[Any, ...]:
    """(codes, validity, type, dictionary) of MIN / MAX of a string column with dictionary ``d`` from MIN / MAX of its
    ranks (``sort.string_ranks``) and the count of its valid rows."""
    return S.codes_of_ranks(d, ranks), (count > 0).to(torch.uint8), tp, d


def m2_of(dev: torch.Tensor, dev2: torch.Tensor, count: torch.Tensor) -> torch.Tensor:
    """M2 = sum of (x - mean)^2 from K6's sums of deviations from a pilot value: DEV2 - DEV^2 / m, clamped at 0
    (float64; ``count`` m as float64)."""
    return torch.clamp_min(dev2 - dev * dev / count, 0.0)


def variance_of(fn: str, m2: torch.Tensor, count: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``fn`` (a ``VARIANCES`` head) from M2 and the non-NULL count m: (float64 values, validity).  The sample
    forms divide by m - 1 and are NULL when m < 2, the population forms divide by m and are NULL when m = 0."""
    samp = fn in ("VAR_SAMP", "STDDEV_SAMP")
    has = count > (1 if samp else 0)
    v = m2 / torch.where(has, count - (1 if samp else 0), torch.ones_like(count)).to(torch.float64)
    if fn.startswith("STDDEV"):
        v = torch.sqrt(v)
    return torch.where(has, v, torch.zeros_like(v)).contiguous(), has.to(torch.uint8)


def shape_moments(gaggs: Sequence[torch.Tensor], slots: Tuple[int, ...]) -> Tuple[torch.Tensor, ...]:
    """(m, M2, M3, M4) per group from the K6 accumulators ``slots`` of a column: SUM, COUNT, DEV, DEV2, DEV3, DEV4,
    MIN, MAX.  DEV .. DEV4 are the sums of d^k, d = x - c, about the atomically summed mean c; with delta = DEV / m
    the central sums are exactly M2 = DEV2 - m delta^2, M3 = DEV3 - 3 delta DEV2 + 2 m delta^3 and
    M4 = DEV4 - 4 delta DEV3 + 6 delta^2 DEV2 - 3 m delta^4 (M2 and M4 clamped at 0).  A column whose MIN equals its
    MAX is constant: all three are exactly 0.  A MIN or MAX that is not finite (a NaN or +-inf) makes all three NaN."""
    _, m, d1, d2, d3, d4, mn, mx = (gaggs[i] for i in slots)
    d1, d2, d3, d4, mn, mx = (q.view(torch.float64) for q in (d1, d2, d3, d4, mn, mx))
    mf = m.to(torch.float64)
    delta = d1 / mf
    dd = delta * delta
    m2 = torch.clamp_min(d2 - mf * dd, 0.0)
    m3 = d3 - 3.0 * delta * d2 + 2.0 * mf * dd * delta
    m4 = torch.clamp_min(d4 - 4.0 * delta * d3 + 6.0 * dd * d2 - 3.0 * mf * dd * dd, 0.0)
    const = mn == mx
    finite = torch.isfinite(mn) & torch.isfinite(mx)
    zero, nan = torch.zeros_like(mf), torch.full_like(mf, math.nan)
    return (m, *(torch.where(finite, torch.where(const, zero, v), nan) for v in (m2, m3, m4)))


def shape_of(fn: str, m: torch.Tensor, m2: torch.Tensor, m3: torch.Tensor,
             m4: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``fn`` (a ``SHAPES`` head) from the non-NULL count m and the central sums M2, M3, M4: (float64 values,
    validity).  SKEWNESS (pandas ``skew()``) is NULL when m < 3, KURTOSIS (pandas ``kurt()``, excess) when m < 4, the
    population forms when m = 0.  M2 = 0 (a constant column) gives 0; a NaN M2 gives NaN."""
    need = {"SKEWNESS": 3, "KURTOSIS": 4}.get(fn, 1)
    has = m >= need
    mf = torch.where(has, m, torch.full_like(m, need)).to(torch.float64)
    flat = m2 == 0
    s2 = torch.where(flat, torch.ones_like(m2), m2)
    if fn.startswith("SKEWNESS"):
        w = mf * torch.sqrt(mf - 1.0) / (mf - 2.0) if fn == "SKEWNESS" else torch.sqrt(mf)
        v = w * m3 / (s2 * torch.sqrt(s2))
    else:
        g = mf * m4 / (s2 * s2)
        if fn == "KURTOSIS":
            den = (mf - 2.0) * (mf - 3.0)
            v = ((mf + 1.0) * (mf - 1.0) * g - 3.0 * (mf - 1.0) * (mf - 1.0)) / den
        else:
            v = g - 3.0
    v = torch.where(flat, torch.zeros_like(v), v)
    return torch.where(has, v, torch.zeros_like(v)).contiguous(), has.to(torch.uint8)


def ewm_of(fn: str, m: torch.Tensor, mean: torch.Tensor, w: torch.Tensor, w2: torch.Tensor, c: torch.Tensor, bias: bool,
           min_periods: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``fn`` (an ``EWM_HEADS`` head) from the running observation count m, weighted mean, W, W2 and C of
    ``fb_segmented_ewm``: (float64 values, validity).  NULL before the first observation and while m < min_periods.
    EWM_VAR is C / W, times W^2 / (W^2 - W2) unless ``bias``, as pandas computes it, and NULL where W^2 - W2 <= 0
    (one observation); EWM_STD is its square root."""
    has = m >= max(min_periods, 1)
    if fn == "EWM_MEAN":
        v = mean
    else:
        ws = torch.where(has, w, torch.ones_like(w))
        v = c / ws
        if not bias:
            num = ws * ws
            den = num - w2
            has = has & (den > 0)
            v = num / torch.where(den > 0, den, torch.ones_like(den)) * v
        if fn == "EWM_STD":
            v = torch.sqrt(v)
    return torch.where(has, v, torch.zeros_like(v)).contiguous(), has.to(torch.uint8)


def pair_moments(gaggs: Sequence[torch.Tensor], slots: Tuple[int, ...]) -> Tuple[torch.Tensor, ...]:
    """(m, mean x, mean y, Sxx, Syy, Sxy) per group from the 12 K6 accumulators of a pair: the corrected two-pass
    DEV2 - DEV^2 / m (clamped at 0) and CODEV - DEVx DEVy / m.  A column whose MIN equals its MAX is constant:
    its S is exactly 0 and so is Sxy (the mean summed with atomics is not exactly the constant).  A NaN or
    +-inf on either side (a MIN or MAX that is not finite) makes all three NaN."""
    sx, sy, cnt, dx, d2x, cod, dy, d2y, mnx, mxx, mny, mxy = (gaggs[i] for i in slots)
    f = [q.view(torch.float64) for q in (sx, sy, dx, d2x, cod, dy, d2y, mnx, mxx, mny, mxy)]
    sx, sy, dx, d2x, cod, dy, d2y, mnx, mxx, mny, mxy = f
    m = cnt
    mf = m.to(torch.float64)
    zero = torch.zeros_like(mf)
    cx, cy = mnx == mxx, mny == mxy
    sxx = torch.where(cx, zero, m2_of(dx, d2x, mf))
    syy = torch.where(cy, zero, m2_of(dy, d2y, mf))
    sxy = torch.where(cx | cy, zero, cod - dx * dy / mf)
    finite = torch.isfinite(mnx) & torch.isfinite(mxx) & torch.isfinite(mny) & torch.isfinite(mxy)
    nan = torch.full_like(mf, math.nan)
    return (m, sx / mf, sy / mf, torch.where(finite, sxx, nan), torch.where(finite, syy, nan),
            torch.where(finite, sxy, nan))


def bivariate_of(fn: str, m: torch.Tensor, mx: torch.Tensor, my: torch.Tensor, sxx: torch.Tensor, syy: torch.Tensor,
                 sxy: torch.Tensor) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """``fn`` (a ``BIVARIATES`` head) from the pair count m, the means of x and y and Sxx, Syy, Sxy over the pair
    rows: (values, validity or None).  REGR_COUNT is m (int64, never NULL); COVAR_SAMP is NULL when m < 2; every
    other function is NULL when m = 0, and SLOPE / INTERCEPT / R2 also when Sxx = 0, CORR when Sxx = 0 or Syy = 0.
    CORR is clamped to [-1, 1] and R2 to [0, 1] (1 when Syy = 0).  A NaN Sxx or Syy is not 0: the result is NaN."""
    if fn == "REGR_COUNT":
        return m.contiguous(), None
    has = m > (1 if fn == "COVAR_SAMP" else 0)
    mf = m.to(torch.float64)
    if fn in ("COVAR_POP", "COVAR_SAMP"):
        v = sxy / torch.where(has, mf - (1 if fn == "COVAR_SAMP" else 0), torch.ones_like(mf))
    elif fn in ("REGR_AVGX", "REGR_AVGY", "REGR_SXX", "REGR_SYY", "REGR_SXY"):
        v = {"REGR_AVGX": mx, "REGR_AVGY": my, "REGR_SXX": sxx, "REGR_SYY": syy, "REGR_SXY": sxy}[fn]
    elif fn == "CORR":
        has = has & (sxx != 0) & (syy != 0)
        v = torch.clamp(sxy / (torch.sqrt(sxx) * torch.sqrt(syy)), -1.0, 1.0)
    else:
        has = has & (sxx != 0)
        slope = sxy / sxx
        if fn == "REGR_SLOPE":
            v = slope
        elif fn == "REGR_INTERCEPT":
            v = my - slope * mx
        else:  # REGR_R2
            v = torch.where(syy == 0, torch.ones_like(syy), torch.clamp(sxy * sxy / (sxx * syy), 0.0, 1.0))
    return torch.where(has, v, torch.zeros_like(v)).contiguous(), has.to(torch.uint8)
