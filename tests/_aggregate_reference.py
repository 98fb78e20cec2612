"""The exact value of every ``column.AGGREGATES`` head over one group, in plain Python.  Test infrastructure only.

Values enter as the engine reduces them (:func:`canonical`): float types as float64 (every float16 / float32 value
widens exactly, a NaN's sign and payload bits kept), strings as ``str``, everything else as its signed 64-bit storage
integer (bool 0 / 1, dates in days or milliseconds, timestamps in their unit).  A uint64 value >= 2^63 is that
integer's bit pattern, negative (DESIGN §7e): SUM, AVG, MIN, MAX and the variances, shape statistics and pair
functions read it so; PERCENTILE_DISC / _CONT order it as unsigned, as the quantile kernel does.

* SUM of integers: the exact sum mod 2^64 (int64); of floats ``oracle.groupby._fsum`` (``math.fsum``, IEEE rules
  for NaN and +-inf, an exact sum beyond the double range is the infinity of its sign).
* AVG: the float64 sum of the values, each widened to float64 as the engine widens it, over the count.
* MIN / MAX: floats in IEEE totalOrder on their float64 bits (``-NaN < -inf < ... < -0.0 < +0.0 < ... < +NaN``),
  the input's own bits; strings by code point; the rest signed.
* FIRST / LAST: the first / last non-NULL value in input row order.
* PERCENTILE_DISC / _CONT: ``oracle.quantile`` (a NaN is NULL, -0.0 ties with 0.0, ties in row order).
* The variances, shape statistics and pair functions: ``oracle.moments``, ``oracle.shape_moments`` and
  ``oracle.comoments`` over exact fractions, rounded once; but REGR_AVGX / REGR_AVGY are AVG of their side over the
  pair rows (DESIGN §7k: the averages follow AVG).

A result is ``None`` for NULL; :data:`REJECTED` for a (function, type) that the engine refuses; :data:`OVERFLOW`
for a variance, shape statistic or pair function (but REGR_COUNT and the averages) of values so large that the float64 power sums of the engine's
algorithms overflow (|x| >= 2^511, or 2^255 for the fourth powers of a shape statistic): no finite value is right
there, as no float64 sum of d^2 (d^4) can hold it.
"""
import math
from typing import Any, List, Optional, Sequence

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from fugue_b200.column import AGGREGATES
from oracle import comoments as OC
from oracle import groupby as og
from oracle import moments as OM
from oracle import quantile as OQ
from oracle import shape_moments as OS

REJECTED = "rejected"
OVERFLOW = "overflow"
_MASK64 = (1 << 64) - 1


def is_string(tp: pa.DataType) -> bool:
    return pa.types.is_string(tp) or pa.types.is_large_string(tp)


def _storage(tp: pa.DataType) -> np.dtype:
    if pa.types.is_floating(tp):
        return np.dtype({16: "f2", 32: "f4", 64: "f8"}[tp.bit_width])
    if pa.types.is_integer(tp):
        return np.dtype(("i" if pa.types.is_signed_integer(tp) else "u") + str(tp.bit_width // 8))
    if pa.types.is_date32(tp):
        return np.dtype("i4")
    if pa.types.is_date64(tp) or pa.types.is_timestamp(tp):
        return np.dtype("i8")
    raise NotImplementedError(tp)


def _f64_of(raw: np.ndarray) -> List[float]:
    """float16 / float32 / float64 values as float64, exactly: a NaN keeps its sign and its payload bits as they
    are (a signalling NaN stays one)."""
    x = raw.astype(np.float64).tolist()
    if raw.dtype != np.float64:
        mbits, width = (10, 16) if raw.dtype == np.float16 else (23, 32)
        u = raw.view(np.uint16 if width == 16 else np.uint32)
        for i in np.flatnonzero(np.isnan(raw)).tolist():
            b = int(u[i])
            x[i] = og.float_of(((b >> (width - 1)) << 63) | (0x7FF << 52) | ((b & ((1 << mbits) - 1)) << (52 - mbits)))
    return x


def canonical(arr: Any) -> List[Any]:
    """The values of an Arrow array (or chunked array) as the engine reduces them; ``None`` for NULL."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    tp = arr.type
    if pa.types.is_dictionary(tp):
        arr = arr.cast(tp.value_type)
        tp = arr.type
    if is_string(tp):
        return arr.to_pylist()
    valid = np.asarray(arr.is_valid()).tolist() if len(arr) else []
    if pa.types.is_boolean(tp):
        x: Any = np.asarray(pc.cast(arr, pa.uint8()).fill_null(0)).astype(np.int64).tolist()
    else:
        st = _storage(tp)
        raw = np.frombuffer(arr.buffers()[1], dtype=st, count=len(arr) + arr.offset)[arr.offset:]
        if st.kind == "f":
            x = _f64_of(raw)
        else:
            x = [og.signed64(int(v)) for v in raw.tolist()]
    return [v if ok else None for v, ok in zip(x, valid)]


def bits(x: float) -> int:
    return og.bits_of(x)


def rejects(fn: str, tp: pa.DataType) -> bool:
    """Whether the engine refuses ``fn`` of an argument of type ``tp``: the variances, the shape statistics and the
    pair functions take integer and float columns only, PERCENTILE_CONT the same, SUM and AVG no strings."""
    family = AGGREGATES[fn].family
    numeric = pa.types.is_integer(tp) or pa.types.is_floating(tp)
    if family in ("variance", "shape", "bivariate") or fn == "PERCENTILE_CONT":
        return not numeric
    return fn in ("SUM", "AVG") and is_string(tp)


def _present(values: Sequence[Any]) -> List[Any]:
    return [v for v in values if v is not None]


def _min_max(fn: str, vals: List[Any], floating: bool) -> Any:
    if floating:
        key = lambda v: og.total_order_key(bits(v))  # noqa: E731
    else:
        key = None
    return min(vals, key=key) if fn == "MIN" else max(vals, key=key)


def _quantile_order(vals: List[Any], tp: pa.DataType) -> List[Any]:
    """The non-NULL, non-NaN values in ascending order, ties in row order."""
    if pa.types.is_floating(tp):
        return sorted((v for v in vals if not math.isnan(v)))
    if pa.types.is_unsigned_integer(tp):
        return sorted(vals, key=lambda v: v & _MASK64)
    return sorted(vals)


def _too_big(vals: Sequence[float], limit: float) -> bool:
    return all(math.isfinite(v) for v in vals) and any(abs(v) >= limit for v in vals)


def _or_overflow(result: Any, big: bool) -> Any:
    """``result()``, but :data:`OVERFLOW` for a non-NULL result of values that are ``big``."""
    try:
        r = result()
    except OverflowError:  # an exact M2 beyond the double range
        assert big
        return OVERFLOW
    return OVERFLOW if big and r is not None else r


def sum_bound(values: Sequence[Any]) -> float:
    """``(m - 1) * 2^-52 * sum(|v|)`` of the non-NULL values as float64: how far an fp64 sum in any order may lie
    from the correctly rounded one (``inf`` when that sum overflows)."""
    vals = [float(v) for v in _present(values)]
    try:
        s = math.fsum(abs(v) for v in vals) if all(math.isfinite(v) for v in vals) else math.inf
    except OverflowError:
        s = math.inf
    return max(len(vals) - 1, 0) * 2.0 ** -52 * s


def aggregate(fn: str, tp: pa.DataType, values: Sequence[Any], q: Optional[float] = None,
              ys: Optional[Sequence[Any]] = None) -> Any:
    """``fn`` over one group: ``values`` (and, for a pair function, ``ys`` of the same rows: x is ``values``, y
    is ``ys``) in input row order, as :func:`canonical` gives them, of arrow type ``tp``.  COUNT counts the
    non-NULL values; ``q`` is the percentile's fraction."""
    if rejects(fn, tp):
        return REJECTED
    family = AGGREGATES[fn].family
    floating = pa.types.is_floating(tp)
    if family == "bivariate":
        pairs = OC.pair_rows([None if v is None else float(v) for v in values],
                             [None if v is None else float(v) for v in ys])
        if fn in ("REGR_AVGX", "REGR_AVGY"):  # the averages follow AVG (DESIGN §7k), overflow of the sum included
            return aggregate("AVG", pa.float64(), [p[0 if fn == "REGR_AVGX" else 1] for p in pairs])
        big = fn != "REGR_COUNT" and _too_big([v for p in pairs for v in p], 2.0 ** 511)
        return _or_overflow(lambda: OC.result_of_state(fn, OC.exact_state(pairs)), big)
    vals = _present(values)
    if fn == "COUNT":
        return len(vals)
    if family == "pick":
        return (vals[0] if fn == "FIRST" else vals[-1]) if vals else None
    if family == "percentile":
        order = _quantile_order(vals, tp)
        if fn == "PERCENTILE_DISC":
            p = OQ.disc_position(len(order), q)
            return None if p is None else order[p]
        x = np.array([float(v & _MASK64) if pa.types.is_unsigned_integer(tp) else float(v) for v in order],
                     dtype=np.float64)
        return OQ.cont(x, q)
    if family == "variance":
        f = [float(v) for v in vals]
        return _or_overflow(lambda: OM.result_exact(fn, f), _too_big(f, 2.0 ** 511))
    if family == "shape":
        f = [float(v) for v in vals]
        return _or_overflow(lambda: OS.result(fn, f), _too_big(f, 2.0 ** 255))
    if not vals:
        return None
    if fn in ("MIN", "MAX"):
        return _min_max(fn, vals, floating)
    if fn == "SUM":
        if floating:
            return og._fsum(np.array(vals, dtype=np.float64))
        return og.signed64(sum(vals))
    assert fn == "AVG", fn
    return og._fsum(np.array([float(v) for v in vals], dtype=np.float64)) / len(vals)

