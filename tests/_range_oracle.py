"""Value frames (``over(range=(start, end))``, RANGE BETWEEN) restated in numpy for the tests: what
``fb_window_range_bounds`` and ``fb_window_bounded`` compute, and whole ``ColumnMap`` results with range nodes.
Test infrastructure only.

Semantics (DESIGN §4).  A logical partition is one PartitionSpec key tuple; its rows are in presort order, NULL
keys last whether the presort is ASC or DESC; a float NaN key is NULL and -0.0 equals 0.0.  For a row i with a
non-NULL key k_i, a row j of its partition with a non-NULL key k_j is in i's frame exactly when

    ASC:  k_i + start <= k_j <= k_i + end          DESC:  k_i - end <= k_j <= k_i - start

with exact mathematical sums for integer, unsigned and temporal keys (no wrap, no saturation: a bound past the
type's range selects nothing on that side; uint64 keys compare as unsigned) and one IEEE f64 addition for float
keys widened to f64 (``+inf - 7 == +inf``; a finite sum that overflows is +-inf).  A NULL key is at distance 0
from the other NULL keys and infinitely far from every value: a NULL-key row's frame is its NULL peers on every
side with an offset or CURRENT ROW, a non-NULL row's frame holds a NULL-key row only through an UNBOUNDED side,
and an UNBOUNDED side runs to the partition's first or last row.  CURRENT ROW is the offset 0: the row's peers.
A frame whose bounds are only CURRENT ROW / UNBOUNDED takes its peers over all presort columns (without a presort
every row of the partition is a peer); a frame with an offset needs exactly one numeric or temporal presort
column.  Aggregation is that of ROWS frames (tests/_frame_oracle.py): NULL-skipping, an empty frame gives NULL
(COUNT 0), integer SUM wraps, float MIN / MAX use IEEE totalOrder and return the input's own bits, FIRST / LAST
take the first / last valid row of the frame.

:func:`range_bounds` is the bounds kernel's contract, :func:`bounded_aggregate` the aggregate kernel's,
:func:`window_map` a whole map: range nodes here, every other node by ``tests/_frame_oracle.window_map``.
"""
import datetime
import math
from collections import OrderedDict
from typing import Any, Dict, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

import _frame_oracle as F
from fugue_b200.column import ColumnExpr, Kind, col
from oracle import expressions as ox
from oracle import sort as S
from oracle import window as W
from oracle.window import _total_order

_LOOP_MAX = 2_000  # rows up to which the plain loops run (they are O(rows x frame))
_I64 = (-(1 << 63), (1 << 63) - 1)
_U64 = (0, (1 << 64) - 1)


def _run_ends(offsets: np.ndarray, valid: np.ndarray) -> np.ndarray:
    """Per segment, the first NULL-key row (its NULL keys are its tail)."""
    bad = np.flatnonzero(~valid)
    j = np.searchsorted(bad, offsets[:-1], "left")
    first_bad = np.append(bad, np.iinfo(np.int64).max)[j]
    return np.minimum(first_bad, offsets[1:])


def _key_list(keys: np.ndarray, cls: str) -> list:
    if cls == "F64":
        return np.asarray(keys, dtype=np.float64).tolist()
    if cls == "U64":
        return np.asarray(keys).view(np.uint64).tolist()
    return np.asarray(keys).view(np.int64).tolist()


def range_bounds(offsets: np.ndarray, keys: np.ndarray, valid: Optional[np.ndarray], cls: str, ascending: bool,
                 start: Any, end: Any, loop: Optional[bool] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Per row, the first and last row of its RANGE frame (last < first: empty), with lo = the first row of the
    non-NULL run at or past the lower bound and hi = the last row at or before the upper bound, as the kernel
    reports them.  ``keys``: int64 (``cls`` "I64"), uint64 bit patterns ("U64") or float64 ("F64") in presort
    order; ``valid``: False for NULL (and NaN) keys, which are each segment's tail."""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = int(offsets[-1])
    ok = np.ones(n, dtype=bool) if valid is None else np.asarray(valid).astype(bool)
    if cls == "F64":
        ok = ok & ~np.isnan(np.asarray(keys, dtype=np.float64))
    lengths = np.diff(offsets)
    first = np.repeat(offsets[:-1], lengths)
    last = np.repeat(offsets[1:] - 1, lengths)
    run_end = np.repeat(_run_ends(offsets, ok), lengths)
    if loop if loop is not None else n <= _LOOP_MAX:
        return _bounds_loop(keys, ok, first, last, run_end, cls, ascending, start, end)
    return _bounds_vec(offsets, keys, ok, first, last, run_end, cls, ascending, start, end)


def _bounds_loop(keys, ok, first, last, run_end, cls, ascending, start, end):
    n = len(ok)
    k = _key_list(keys, cls)
    lo = np.zeros(n, dtype=np.int64)
    hi = np.zeros(n, dtype=np.int64)

    def bound(x: Any, off: Any, sign: int) -> Any:
        if cls == "F64":
            with np.errstate(over="ignore"):
                return float(np.float64(x) + np.float64(sign * float(off)))  # one IEEE addition
        return x + sign * int(off)  # python ints: exact

    for i in range(n):
        a, b, e = int(first[i]), int(last[i]) + 1, int(run_end[i])
        if not ok[i]:
            lo[i] = a if start is None else e
            hi[i] = b - 1
            continue
        run = k[a:e]
        if start is None:
            lo[i] = a
        elif ascending:  # rows below k_i + start come first
            t = bound(k[i], start, 1)
            lo[i] = a + sum(1 for x in run if x < t)
        else:  # rows above k_i - start come first
            t = bound(k[i], start, -1)
            lo[i] = a + sum(1 for x in run if x > t)
        if end is None:
            hi[i] = b - 1
        elif ascending:
            t = bound(k[i], end, 1)
            hi[i] = a - 1 + sum(1 for x in run if x <= t)
        else:
            t = bound(k[i], end, -1)
            hi[i] = a - 1 + sum(1 for x in run if x >= t)
    return lo, hi


def _bounds_vec(offsets, keys, ok, first, last, run_end, cls, ascending, start, end):
    """Every segment's non-NULL run searched at once: a run sorted by dense value rank, prefixed by its segment."""
    n = len(ok)
    seg = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    if cls == "F64":
        k = np.asarray(keys, dtype=np.float64)
    else:
        k = np.asarray(keys).view(np.uint64 if cls == "U64" else np.int64)
    uniq = np.unique(k[ok])
    u = len(uniq)
    rank = np.searchsorted(uniq, k[ok], "left")
    if not ascending:
        rank = u - 1 - rank
    comb = seg[ok].astype(np.int64) * (u + 1) + rank  # ascending over the runs, in row order
    base = np.searchsorted(comb, seg.astype(np.int64) * (u + 1), "left")

    def below(cut: np.ndarray) -> np.ndarray:  # rows of i's run whose rank is below cut
        return np.searchsorted(comb, seg.astype(np.int64) * (u + 1) + cut, "left") - base

    def cuts(off: Any, sign: int) -> Tuple[np.ndarray, np.ndarray]:
        """(#values < t, #values <= t) among uniq for every row's t = k + sign * off, exactly."""
        if cls == "F64":
            with np.errstate(over="ignore"):
                t = k + np.float64(sign * float(off))
            return np.searchsorted(uniq, t, "left"), np.searchsorted(uniq, t, "right")
        o = sign * int(off)
        lo_t, hi_t = _U64 if cls == "U64" else _I64
        with np.errstate(over="ignore"):
            if cls == "U64" and abs(o) < (1 << 64):  # wrapping uint64 arithmetic, the carry read off the result
                m = np.uint64(abs(o))
                t = k + m if o >= 0 else k - m
                big = (t < k) if o >= 0 else np.zeros(len(k), dtype=bool)
                small = (k < m) if o < 0 else np.zeros(len(k), dtype=bool)
            elif cls == "I64" and lo_t <= o <= hi_t:
                t = k + np.int64(o)
                big = (t < k) if o > 0 else np.zeros(len(k), dtype=bool)
                small = (t > k) if o < 0 else np.zeros(len(k), dtype=bool)
            else:  # python ints
                x = [v + o for v in k.tolist()]
                big = np.array([v > hi_t for v in x], dtype=bool)
                small = np.array([v < lo_t for v in x], dtype=bool)
                t = np.array([min(max(v, lo_t), hi_t) for v in x], dtype=k.dtype)
        sl, sr = np.searchsorted(uniq, t, "left"), np.searchsorted(uniq, t, "right")
        sl = np.where(big, u, np.where(small, 0, sl))
        sr = np.where(big, u, np.where(small, 0, sr))
        return sl, sr

    a = first
    if start is None:
        lo = first.copy()
    else:
        sl, sr = cuts(start, 1 if ascending else -1)
        lo = a + below(sl if ascending else u - sr)
    if end is None:
        hi = last.copy()
    else:
        sl, sr = cuts(end, 1 if ascending else -1)
        hi = a - 1 + below(sr if ascending else u - sl)
    lo = np.where(ok, lo, first if start is None else run_end)
    hi = np.where(ok, hi, last)
    return lo.astype(np.int64), hi.astype(np.int64)


def bounded_aggregate(values: Optional[np.ndarray], valid: Optional[np.ndarray], lo: np.ndarray, hi: np.ndarray,
                      op: str, loop: Optional[bool] = None) -> Tuple[Optional[np.ndarray], np.ndarray]:
    """``op`` (as in ``oracle.window.segmented_scan``) over the valid rows of ``[lo[i], hi[i]]`` clamped to the
    table (hi < lo: empty).  Returns (values or None for COUNT, counts), the value 0 where the count is 0.  The
    loop adds a SUM_F64 frame with ``math.fsum``; the vectorised form is exact for COUNT, SUM_I64 and MIN / MAX
    (a sparse table) and takes SUM_F64 as a prefix-sum difference, exact whenever every partial sum is."""
    lo = np.asarray(lo, dtype=np.int64)
    hi = np.asarray(hi, dtype=np.int64)
    n = len(lo)
    ok = np.ones(n, dtype=bool) if valid is None else np.asarray(valid).astype(bool)
    v = None if values is None else np.asarray(values).view(np.int64)
    a_ = np.clip(lo, 0, n)
    b_ = np.clip(hi, -1, n - 1) + 1 if n else np.zeros(0, np.int64)  # clipped before the + 1: no overflow
    b_ = np.maximum(a_, b_)
    if loop if loop is not None else n <= _LOOP_MAX:
        out = np.zeros(n, dtype=np.int64)
        cnt = np.zeros(n, dtype=np.int64)
        for i in range(n):
            sel = np.arange(a_[i], b_[i])
            sel = sel[ok[sel]]
            cnt[i] = len(sel)
            if len(sel) == 0 or op == "COUNT":
                continue
            x = v[sel]
            if op == "SUM_I64":
                out[i] = ((sum(int(y) for y in x) + 2**63) % 2**64) - 2**63
            elif op == "SUM_F64":
                out[i] = np.float64(math.fsum(x.view(np.float64).tolist())).view(np.int64)
            else:
                key = _total_order(x) if op.endswith("F64") else x
                out[i] = x[int(np.argmin(key) if op.startswith("MIN") else np.argmax(key))]
        return (None if op == "COUNT" else out), cnt
    cs = np.concatenate([np.zeros(1, np.int64), np.cumsum(ok.astype(np.int64))])
    cnt = cs[b_] - cs[a_]
    if op == "COUNT":
        return None, cnt
    if op == "SUM_I64":
        p = np.concatenate([np.zeros(1, np.uint64), np.cumsum(np.where(ok, v, 0).view(np.uint64), dtype=np.uint64)])
        out = (p[b_] - p[a_]).view(np.int64)
    elif op == "SUM_F64":
        p = np.concatenate([np.zeros(1), np.cumsum(np.where(ok, v.view(np.float64), 0.0))])
        out = (p[b_] - p[a_]).view(np.int64)
    else:
        is_f, mn = op.endswith("F64"), op.startswith("MIN")
        fill = np.iinfo(np.int64).max if mn else np.iinfo(np.int64).min
        x = np.where(ok, _total_order(v) if is_f else v, fill)
        table = [x]
        while (1 << len(table)) <= n:
            prev, h = table[-1], 1 << (len(table) - 1)
            table.append(np.minimum(prev[:-h], prev[h:]) if mn else np.maximum(prev[:-h], prev[h:]))
        width = np.maximum(b_ - a_, 1)
        lev = np.floor(np.log2(width)).astype(np.int64)
        lev = np.where((1 << (lev + 1)) <= width, lev + 1, lev)  # guard the float log
        lev = np.where((1 << lev) > width, lev - 1, lev)
        out = np.zeros(n, dtype=np.int64)
        for l_ in np.unique(lev).tolist():
            m = (lev == l_) & (cnt > 0)
            t = table[l_]
            left = t[a_[m]]
            right = t[b_[m] - (1 << l_)]
            red = np.minimum(left, right) if mn else np.maximum(left, right)
            out[m] = _total_order(red) if is_f else red
    return np.where(cnt > 0, out, 0), cnt


# ---- whole maps -----------------------------------------------------------------------------------
_UNIT_US = {"s": 1_000_000, "ms": 1_000, "us": 1, "D": 86_400_000_000}


def _presort_key(st: pa.Table, name: str) -> Tuple[np.ndarray, np.ndarray, str, Optional[str]]:
    """(key values, validity, class, time unit) of the presort column in the sorted table."""
    a = st.column(name).combine_chunks()
    tp = a.type
    ok = np.ones(len(a), dtype=bool) if a.null_count == 0 else np.asarray(pc.is_valid(a).to_numpy(zero_copy_only=False))
    if pa.types.is_floating(tp):
        k = np.asarray(a.cast(pa.float64()).fill_null(0).to_numpy(zero_copy_only=False), dtype=np.float64)
        return k, ok & ~np.isnan(k), "F64", None
    if pa.types.is_unsigned_integer(tp):
        return np.asarray(a.cast(pa.uint64()).fill_null(0).to_numpy(zero_copy_only=False)), ok, "U64", None
    if pa.types.is_integer(tp):
        return np.asarray(a.cast(pa.int64()).fill_null(0).to_numpy(zero_copy_only=False)), ok, "I64", None
    unit = "D" if pa.types.is_date32(tp) else ("ms" if pa.types.is_date64(tp) else tp.unit)
    storage = pa.int32() if pa.types.is_date32(tp) else pa.int64()
    ints = a.view(storage).cast(pa.int64()).fill_null(0)
    return np.asarray(ints.to_numpy(zero_copy_only=False)), ok, "I64", unit


def _offset(b: Any, cls: str, unit: Optional[str]) -> Any:
    if b is None or cls == "F64":
        return None if b is None else float(b)
    if isinstance(b, datetime.timedelta):
        us = b // datetime.timedelta(microseconds=1)
        if unit == "ns":
            return us * 1000
        assert us % _UNIT_US[unit] == 0
        return us // _UNIT_US[unit]
    return int(b)


def _range_column(e: ColumnExpr, st: pa.Table, pdf: Any, offsets: np.ndarray, presort: "OrderedDict[str, bool]",
                  seg_head: np.ndarray) -> pa.Array:
    """One range node ``e`` (no alias, no cast) over the sorted table ``st``, in its row order."""
    fn = e.func
    start, end = e.kwargs["range"]
    n = st.num_rows
    lengths = np.diff(offsets)
    if all(b is None or b == 0 for b in (start, end)):  # peers over every presort column
        peer = S.group_heads(st, list(presort.keys())) | seg_head
        pos = np.arange(n, dtype=np.int64)
        peer_first = np.maximum.accumulate(np.where(peer, pos, 0)) if n else pos
        nxt = np.append(peer[1:], True) if n else peer
        peer_last = np.minimum.accumulate(np.where(nxt, pos, n)[::-1])[::-1] if n else pos
        lo = np.repeat(offsets[:-1], lengths) if start is None else peer_first
        hi = np.repeat(offsets[1:] - 1, lengths) if end is None else peer_last
    else:
        (name, asc), = presort.items()
        k, ok, cls, unit = _presort_key(st, name)
        lo, hi = range_bounds(offsets, k, ok, cls, asc, _offset(start, cls, unit), _offset(end, cls, unit))

    def agg(x: Optional[np.ndarray], ok_: Optional[np.ndarray], op: str) -> Tuple[Any, np.ndarray]:
        return bounded_aggregate(x, ok_, lo, hi, op)

    if e.arg.kind == Kind.WILDCARD:
        return pa.array(agg(None, None, "COUNT")[1], type=pa.int64())
    if e.arg.kind == Kind.NAMED and e.arg.as_type is None:
        v, ok, tp = W._column(st, e.arg.name)
    else:
        v, ok, tp = W._column(pa.table({"x": pa.array(ox.evaluate(e.arg, pdf), from_pandas=True)}), "x")
    if fn == "COUNT":
        return pa.array(agg(None, ok, "COUNT")[1], type=pa.int64())
    if fn in ("FIRST", "LAST"):
        r, c = agg(np.arange(n, dtype=np.int64), ok, "MIN_I64" if fn == "FIRST" else "MAX_I64")
        return pa.array([(v[j] if ok[j] else None) if m > 0 else None for j, m in zip(r.tolist(), c.tolist())],
                        type=tp)
    is_f = pa.types.is_floating(tp)
    if fn in ("SUM", "AVG"):
        f64 = fn == "AVG" or is_f
        x = v.astype(np.float64).view(np.int64) if f64 else v.astype(np.int64)
        r, c = agg(x, ok, "SUM_F64" if f64 else "SUM_I64")
        out = r.view(np.float64) / np.maximum(c, 1) if fn == "AVG" else (r.view(np.float64) if f64 else r)
        return pa.array(out, type=pa.float64() if f64 else pa.int64(), mask=c == 0)
    if fn in ("MIN", "MAX"):
        x = v.astype(np.float64).view(np.int64) if is_f else v.astype(np.int64)
        r, c = agg(x, ok, f"{fn}_{'F64' if is_f else 'I64'}")
        out = r.view(np.float64).astype(tp.to_pandas_dtype()) if is_f else r.astype(tp.to_pandas_dtype())
        return pa.array(out, type=tp, mask=c == 0)
    raise NotImplementedError(fn)


def window_map(table: pa.Table, keys: Sequence[str], presort: "OrderedDict[str, bool]",
               columns: Sequence[ColumnExpr]) -> Dict[str, list]:
    """``_frame_oracle.window_map`` for maps that may hold range nodes: each distinct range node becomes a column
    of the input (computed over the same partitions and presort order), the rest goes to ``_frame_oracle``."""
    n = table.num_rows
    sorts = OrderedDict((k, True) for k in keys)
    for k, a in presort.items():
        sorts[k] = a
    order = S.argsort(table, sorts, "last")
    st = table.take(pa.array(order, type=pa.int64()))
    seg_head = S.group_heads(st, keys)
    offsets = np.concatenate([np.flatnonzero(seg_head), [n]]).astype(np.int64)
    if n == 0:
        offsets = np.array([0, 0], dtype=np.int64)
    seg_head = seg_head if n else np.zeros(0, dtype=bool)
    pdf = W._pandas(st)
    inverse = np.empty(n, dtype=np.int64)
    inverse[order] = np.arange(n)
    temps: Dict[str, pa.Array] = {}

    def replace(e: Any) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if e.kind == Kind.WINDOW and "range" in e.kwargs:
            bare = e.alias("").cast(None)
            uid = "__r" + bare.fingerprint()[:12]
            if uid not in temps:
                temps[uid] = _range_column(bare, st, pdf, offsets, presort, seg_head).take(
                    pa.array(inverse, type=pa.int64()))
            rep = col(uid)
            if e.as_type is not None:
                rep = rep.cast(e.as_type)
            return rep.alias(e.as_name) if e.as_name else rep
        if e.has_args:
            return ColumnExpr(e.kind, e.head, [replace(a) for a in e.args],
                              {k: replace(v) for k, v in e.kwargs.items()}, e.is_distinct, e.as_name, e.as_type)
        return e

    exprs = [replace(c.infer_alias()) for c in columns]
    full = table
    for k, a in temps.items():
        full = full.append_column(k, a)
    return F.window_map(full, keys, presort, exprs)
