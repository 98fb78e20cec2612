"""Oracle: numpy / pandas restatement of the window functions of a ``ColumnMap`` (K9).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) - never imported by the product path.

In the reference a running total, a forward fill, a rank or a row's share of its group is a pandas
function that ``PandasMapEngine.map_dataframe`` calls once per logical partition, after sorting the
partition by the presort (fugue/execution/native_execution_engine.py:104-169).  This module states what
the window nodes of ``fugue_b200.column`` mean with SQL window semantics over those partitions:

* a logical partition is one distinct key tuple (NULL equal to NULL); rows inside it are in presort order
  (NULLs last in every presort column, ties in input order: a stable sort), in input order without one;
* peers (RANK / DENSE_RANK) are rows equal on every presort column, NULL equal to NULL; without a
  presort every row of a partition is a peer of every other;
* ordering, partitions and peers come from oracle/sort.py, so float keys and presort columns follow its rule:
  a NaN of either sign is NULL, -0.0 equals 0.0 (the rows keep their own bits);
* aggregates skip NULLs; SUM / AVG / MIN / MAX over no valid row are NULL, COUNT never is; FIRST / LAST
  are the first / last valid value; ``running`` = ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW;
* types follow ``ExecutionEngine.aggregate``: integer SUM is int64 with two's-complement wrap-around,
  float SUM and AVG float64, COUNT and the ranks int64, MIN / MAX / FIRST / LAST / LAG / LEAD keep the
  argument's type; float MIN / MAX follow IEEE totalOrder and return the input's own bit pattern.

:func:`segmented_scan` is the scan itself on numpy arrays (what ``fb_segmented_scan`` computes);
:func:`window_map` evaluates a whole ``ColumnMap`` on an Arrow table.
"""
import datetime
import math
import struct
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc

from fugue_b200.column import ColumnExpr, Kind, col

from . import expressions as ox
from . import sort as S

_FLIP = np.int64(0x7FFFFFFFFFFFFFFF)


def _total_order(bits: np.ndarray) -> np.ndarray:
    """int64 bit patterns of doubles -> int64 keys ordered like IEEE totalOrder (an involution)."""
    return np.where(bits >= 0, bits, bits ^ _FLIP)


def segmented_scan(values: Optional[np.ndarray], valid: Optional[np.ndarray], offsets: np.ndarray,
                   op: str) -> Tuple[Optional[np.ndarray], np.ndarray]:
    """Inclusive scan restarting at every ``offsets[s]`` over the rows whose ``valid`` is set.  ``op`` in
    SUM_I64 SUM_F64 MIN_I64 MAX_I64 MIN_F64 MAX_F64 COUNT; values are int64 arrays (the bit patterns for
    the F64 ops).  Returns (values or None for COUNT, counts); the value is 0 where the count is 0."""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = int(offsets[-1])
    lengths = np.diff(offsets)
    starts = offsets[:-1][lengths > 0]
    reps = lengths[lengths > 0]
    seg = np.repeat(np.arange(len(reps)), reps)
    ok = np.ones(n, dtype=bool) if valid is None else np.asarray(valid).astype(bool)
    cs = np.cumsum(ok.astype(np.int64))
    counts = cs - np.repeat((cs - ok)[starts], reps) if n else np.zeros(0, np.int64)
    if op == "COUNT":
        return None, counts
    v = np.asarray(values).view(np.int64)
    if op == "SUM_I64":  # modulo 2^64, exactly: prefix sums in uint64 (numpy wraps) minus the segment's base
        u = np.where(ok, v, 0).view(np.uint64)
        cu = np.cumsum(u, dtype=np.uint64)
        out = (cu - np.repeat((cu - u)[starts], reps)).view(np.int64) if n else v.copy()
    elif op == "SUM_F64":  # row order within a segment
        f = np.where(ok, v.view(np.float64), 0.0)
        out = pd.Series(f).groupby(seg).cumsum().to_numpy(dtype=np.float64).view(np.int64) if n else v.copy()
    elif op in ("MIN_I64", "MAX_I64", "MIN_F64", "MAX_F64"):
        key = _total_order(v) if op.endswith("F64") else v
        lo = op.startswith("MIN")
        sentinel = np.iinfo(np.int64).max if lo else np.iinfo(np.int64).min
        key = np.where(ok, key, sentinel)
        g = pd.Series(key).groupby(seg)
        out = (g.cummin() if lo else g.cummax()).to_numpy(dtype=np.int64) if n else v.copy()
        if op.endswith("F64"):
            out = _total_order(out)
    else:
        raise ValueError(op)
    return np.where(counts > 0, out, 0), counts


# ---- LAG / LEAD defaults ----------------------------------------------------------------------------
_INT_BITS = {pa.int8(): (8, True), pa.int16(): (16, True), pa.int32(): (32, True), pa.int64(): (64, True),
             pa.uint8(): (8, False), pa.uint16(): (16, False), pa.uint32(): (32, False), pa.uint64(): (64, False)}
_PER_UNIT_US = {"D": (86_400_000_000, 1), "s": (1_000_000, 1), "ms": (1000, 1), "us": (1, 1), "ns": (1, 1000)}


def _small_float_bits(x: float, fmt: str, width: int, mbits: int) -> int:
    """``x`` rounded to nearest in the IEEE format of ``width`` bits (``struct`` format ``fmt``); a NaN keeps its
    sign and the top ``mbits`` bits of its payload (the lowest bit set if none is left)."""
    b64 = struct.unpack("<Q", struct.pack("<d", x))[0]
    sign = b64 >> 63
    if math.isnan(x):
        mant = (b64 >> (52 - mbits)) & ((1 << mbits) - 1)
        expo = ((1 << (width - 1 - mbits)) - 1) << mbits
        return (sign << (width - 1)) | expo | (mant or 1)
    try:
        return struct.unpack("<H" if width == 16 else "<I", struct.pack(fmt, x))[0]
    except OverflowError:  # rounds past the largest finite value: the infinity of its sign
        return struct.unpack("<H" if width == 16 else "<I", struct.pack(fmt, math.copysign(math.inf, x)))[0]


def offset_default(d: Any, tp: pa.DataType) -> pa.Array:
    """LAG / LEAD's default as a one-element array of the argument's type, converted as a literal in a CAST to ``tp``:
    floats rounded to nearest once from the float64 value, integers in the type's range, True / False for bool, DATE / TIMESTAMP literals in a
    date or timestamp column's units, a timedelta in a duration's, a string for a string.  ValueError where the type
    cannot hold the default exactly."""
    def bad() -> ValueError:
        return ValueError(f"a LAG / LEAD default {d!r} does not convert exactly to {tp}")

    if pa.types.is_string(tp) or pa.types.is_large_string(tp):
        if not isinstance(d, str):
            raise bad()
        return pa.array([d], type=tp)
    if isinstance(d, str):
        raise bad()
    if pa.types.is_boolean(tp):
        if not isinstance(d, bool):
            raise bad()
        return pa.array([d], type=tp)
    if isinstance(d, bool):
        raise bad()
    if pa.types.is_floating(tp):
        if not isinstance(d, (int, float)):
            raise bad()
        try:
            x = float(d)
        except OverflowError as e:  # an integer past float64
            raise bad() from e
        if tp == pa.float64():
            return pa.array([x], type=tp)
        if tp == pa.float32():
            return pa.array(np.array([_small_float_bits(x, "<f", 32, 23)], np.uint32).view(np.float32))
        return pa.array(np.array([_small_float_bits(x, "<e", 16, 10)], np.uint16).view(np.float16))
    if tp in _INT_BITS:
        if isinstance(d, float) and d.is_integer():
            d = int(d)
        if not isinstance(d, int):
            raise bad()
        bits, signed = _INT_BITS[tp]
        lo, hi = (-(1 << (bits - 1)), 1 << (bits - 1)) if signed else (0, 1 << bits)
        if not lo <= d < hi:
            raise bad()
        return pa.array([d], type=tp)
    span = pa.types.is_duration(tp)
    if pa.types.is_date(tp) or pa.types.is_timestamp(tp) or span:
        if not isinstance(d, (datetime.date, datetime.timedelta)) or span != isinstance(d, datetime.timedelta):
            raise bad()
        if isinstance(d, datetime.timedelta):
            us = d // datetime.timedelta(microseconds=1)
        else:
            dt = d if isinstance(d, datetime.datetime) else datetime.datetime(d.year, d.month, d.day)
            if dt.tzinfo is not None:  # an aware timestamp: its UTC time
                dt = dt.astimezone(datetime.timezone.utc).replace(tzinfo=None)
            us = (dt - datetime.datetime(1970, 1, 1)) // datetime.timedelta(microseconds=1)
        unit = "D" if pa.types.is_date32(tp) else ("ms" if pa.types.is_date64(tp) else tp.unit)
        per, mul = _PER_UNIT_US[unit]
        if (us * mul) % per:
            raise bad()
        v = us * mul // per
        bits = 32 if pa.types.is_date32(tp) else 64
        if not -(1 << (bits - 1)) <= v < (1 << (bits - 1)):
            raise bad()
        return pa.array([v], type=pa.int32() if bits == 32 else pa.int64()).cast(tp)
    raise bad()


# ---- whole maps -----------------------------------------------------------------------------------
def _column(t: pa.Table, name: str) -> Tuple[np.ndarray, np.ndarray, pa.DataType]:
    a = t.column(name).combine_chunks()
    ok = np.ones(len(a), dtype=bool) if a.null_count == 0 else np.asarray(pc.is_valid(a).to_numpy(zero_copy_only=False))
    if pa.types.is_string(a.type) or pa.types.is_large_string(a.type):
        vals = np.array(a.to_pylist(), dtype=object)
    else:
        vals = np.asarray(a.fill_null(0).to_numpy(zero_copy_only=False))
    return vals, ok, a.type


def _pandas(t: pa.Table) -> pd.DataFrame:
    m = {pa.int64(): pd.Int64Dtype(), pa.int32(): pd.Int32Dtype(), pa.float64(): pd.Float64Dtype(),
         pa.float32(): pd.Float32Dtype(), pa.string(): pd.StringDtype(), pa.bool_(): pd.BooleanDtype()}
    return t.to_pandas(types_mapper=m.get)


def window_map(table: pa.Table, keys: Sequence[str], presort: "OrderedDict[str, bool]",
               columns: Sequence[ColumnExpr]) -> Dict[str, list]:
    """Output columns (python values, None for NULL) of ``ColumnMap(*columns)`` under
    ``PartitionSpec(by=keys, presort=presort)``, one entry per input row in input order."""
    n = table.num_rows
    sorts = OrderedDict((k, True) for k in keys)
    for k, a in presort.items():  # a key re-listed in the presort takes the presort's direction, as map_dataframe
        sorts[k] = a
    order = S.argsort(table, sorts, "last")
    st = table.take(pa.array(order, type=pa.int64()))
    seg_head = S.group_heads(st, keys)
    offsets = np.concatenate([np.flatnonzero(seg_head), [n]]).astype(np.int64)
    lengths = np.diff(offsets)
    first = np.repeat(offsets[:-1], lengths)
    last = np.repeat(offsets[1:] - 1, lengths)
    pos = np.arange(n, dtype=np.int64)
    peer = S.group_heads(st, list(presort.keys())) | seg_head
    pdf = _pandas(st)
    temps: Dict[str, pa.Array] = {}

    def arg_of(e: ColumnExpr) -> Tuple[np.ndarray, np.ndarray, pa.DataType]:
        if e.kind == Kind.NAMED and e.as_type is None:
            return _column(st, e.name)
        s = ox.evaluate(e, pdf)
        a = pa.array(s, from_pandas=True)
        return _column(pa.table({"x": a}), "x")

    def window(e: ColumnExpr) -> pa.Array:
        fn = e.func
        if fn == "ROW_NUMBER":
            return pa.array(pos - first + 1, type=pa.int64())
        if fn == "RANK":
            v, _ = segmented_scan(np.where(peer, pos - first + 1, 0), None, offsets, "MAX_I64")
            return pa.array(v, type=pa.int64())
        if fn == "DENSE_RANK":
            v, _ = segmented_scan(peer.astype(np.int64), None, offsets, "SUM_I64")
            return pa.array(v, type=pa.int64())
        if fn in ("LAG", "LEAD"):
            if e.arg.kind == Kind.NAMED and e.arg.as_type is None:
                a = st.column(e.arg.name).combine_chunks()
            else:
                a = pa.array(ox.evaluate(e.arg, pdf), from_pandas=True)
            d = e.kwargs["default"]
            # the source row in python ints, exact for every n >= 0; outside the partition: the appended default
            step = -e.kwargs["n"] if fn == "LAG" else e.kwargs["n"]
            src = [p + step if lo <= p + step <= hi else n for p, lo, hi in zip(range(n), first.tolist(), last.tolist())]
            tail = pa.nulls(1, a.type) if d is None else offset_default(d, a.type)
            return pa.concat_arrays([a, tail]).take(pa.array(src, type=pa.int64()))
        whole = not e.kwargs["running"]

        def fin(x: np.ndarray) -> np.ndarray:
            return x[last] if whole else x

        if e.arg.kind == Kind.WILDCARD:
            _, c = segmented_scan(None, None, offsets, "COUNT")
            return pa.array(fin(c), type=pa.int64())
        v, ok, tp = arg_of(e.arg)
        if fn == "COUNT":
            _, c = segmented_scan(None, ok, offsets, "COUNT")
            return pa.array(fin(c), type=pa.int64())
        if fn in ("FIRST", "LAST"):
            r, c = segmented_scan(pos, ok, offsets, "MIN_I64" if fn == "FIRST" else "MAX_I64")
            r, c = fin(r), fin(c)
            return pa.array([(v[j] if ok[j] else None) if k > 0 else None for j, k in zip(r.tolist(), c.tolist())],
                            type=tp)
        if v.dtype == object:
            raise NotImplementedError(f"{fn} on a string column")
        is_f = pa.types.is_floating(tp)
        if fn in ("SUM", "AVG"):
            f64 = fn == "AVG" or is_f
            x = v.astype(np.float64).view(np.int64) if f64 else v.astype(np.int64)
            r, c = segmented_scan(x, ok, offsets, "SUM_F64" if f64 else "SUM_I64")
            r, c = fin(r), fin(c)
            out = r.view(np.float64) / np.maximum(c, 1) if fn == "AVG" else (r.view(np.float64) if f64 else r)
            return pa.array(out, type=pa.float64() if f64 else pa.int64(), mask=c == 0)
        if fn in ("MIN", "MAX"):
            x = v.astype(np.float64).view(np.int64) if is_f else v.astype(np.int64)
            r, c = segmented_scan(x, ok, offsets, f"{fn}_{'F64' if is_f else 'I64'}")
            r, c = fin(r), fin(c)
            out = r.view(np.float64).astype(tp.to_pandas_dtype()) if is_f else r.astype(tp.to_pandas_dtype())
            return pa.array(out, type=tp, mask=c == 0)
        raise NotImplementedError(fn)

    def replace(e: Any) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if e.kind == Kind.WINDOW:
            bare = e.alias("").cast(None)
            uid = "__w" + bare.fingerprint()[:12]
            if uid not in temps:
                temps[uid] = window(bare)
            rep = col(uid)
            if e.as_type is not None:
                rep = rep.cast(e.as_type)
            return rep.alias(e.as_name) if e.as_name else rep
        if e.has_args:
            return ColumnExpr(e.kind, e.head, [replace(a) for a in e.args],
                              {k: replace(v) for k, v in e.kwargs.items()}, e.is_distinct, e.as_name, e.as_type)
        return e

    exprs = [replace(c.infer_alias()) for c in columns]
    full = st
    for k, a in temps.items():
        full = full.append_column(k, a)
    fdf = _pandas(full)
    inverse = np.empty(n, dtype=np.int64)
    inverse[order] = np.arange(n)
    out: Dict[str, list] = {}
    for e in exprs:
        if e.kind == Kind.NAMED and e.as_type is None:
            vals = full.column(e.name).to_pylist()
        else:
            s = ox.evaluate(e, fdf)
            vals = [None if x is pd.NA or x is None else x for x in s.tolist()]
        out[e.output_name] = [vals[i] for i in inverse.tolist()]
    return out
