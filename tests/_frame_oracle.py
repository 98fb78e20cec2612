"""Moving frames (``over(rows=(start, end))``, ROWS BETWEEN) restated in numpy / pandas for the tests: what
``fb_window_frame`` computes, and whole ``ColumnMap`` results with frame nodes.  Test infrastructure only.

Semantics, extending the statement at the top of oracle/window.py: row i of a logical partition covering rows
[a, b) in presort order aggregates the rows [max(a, i + start), min(b - 1, i + end)], a ``None`` bound clipping to
a or b - 1.  The frame may be empty (``(-3, -1)`` on a partition's first row), which is an aggregate over no valid
row: NULL, COUNT 0.  NULL values are skipped, types follow ``aggregate``, float MIN / MAX follow IEEE totalOrder
and return the input's own bits, integer SUM wraps around, float keys and presort columns follow oracle/sort.py.

:func:`frame_aggregate` is the kernel's contract on numpy arrays; :func:`window_map` evaluates a whole map: frame
nodes here, everything else by ``oracle.window.window_map``.
"""
import math
from collections import OrderedDict
from typing import Any, Dict, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

from fugue_b200.column import ColumnExpr, Kind, col
from oracle import expressions as ox
from oracle import sort as S
from oracle import window as W
from oracle.window import _total_order, segmented_scan


def frame_bounds(offsets: np.ndarray, start: Optional[int], end: Optional[int]) -> Tuple[np.ndarray, np.ndarray]:
    """Per row, the first and last row of its frame (last < first: empty)."""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = int(offsets[-1])
    lengths = np.diff(offsets)
    first = np.repeat(offsets[:-1], lengths)
    last = np.repeat(offsets[1:] - 1, lengths)
    pos = np.arange(n, dtype=np.int64)
    clip = lambda b: min(max(int(b), -n - 1), n + 1)  # noqa: E731 - same frames, no int64 overflow
    lo = first if start is None else np.maximum(first, pos + clip(start))
    hi = last if end is None else np.minimum(last, pos + clip(end))
    return lo, hi


_LOOP_MAX = 20_000  # rows up to which frame_aggregate runs the plain loop


def frame_aggregate(values: Optional[np.ndarray], valid: Optional[np.ndarray], offsets: np.ndarray, op: str,
                    start: Optional[int], end: Optional[int], rows: Optional[np.ndarray] = None,
                    loop: Optional[bool] = None) -> Tuple[Optional[np.ndarray], np.ndarray]:
    """``op`` (as in :func:`segmented_scan`) over the valid rows of every row's frame
    ``ROWS BETWEEN start AND end`` (``None``: UNBOUNDED) inside its segment.  Returns (values or None for
    COUNT, counts), the value 0 where the count is 0; with ``rows``, only those rows, by the loop.

    The loop adds a SUM_F64 frame with ``math.fsum`` (correctly rounded).  The vectorised form (above
    ``_LOOP_MAX`` rows, or ``loop=False``) is exact for COUNT, SUM_I64 (prefix differences mod 2^64) and
    MIN / MAX; its SUM_F64 adds the frame's own values only (a masked window sum, or a running sum in row
    order with an unbounded side), so it is exact whenever every partial sum is."""
    lo, hi = frame_bounds(offsets, start, end)
    n = len(lo)
    ok = np.ones(n, dtype=bool) if valid is None else np.asarray(valid).astype(bool)
    v = None if values is None else np.asarray(values).view(np.int64)
    if rows is not None or (loop if loop is not None else n <= _LOOP_MAX):
        idx = np.arange(n) if rows is None else np.asarray(rows, dtype=np.int64)
        out = np.zeros(len(idx), dtype=np.int64)
        cnt = np.zeros(len(idx), dtype=np.int64)
        for k, i in enumerate(idx.tolist()):
            sel = np.arange(lo[i], hi[i] + 1)
            sel = sel[ok[sel]]
            cnt[k] = len(sel)
            if len(sel) == 0 or op == "COUNT":
                continue
            x = v[sel]
            if op == "SUM_I64":
                out[k] = ((sum(int(a) for a in x) + 2**63) % 2**64) - 2**63
            elif op == "SUM_F64":
                out[k] = np.float64(math.fsum(x.view(np.float64).tolist())).view(np.int64)
            else:
                key = _total_order(x) if op.endswith("F64") else x
                j = int(np.argmin(key) if op.startswith("MIN") else np.argmax(key))
                out[k] = x[j]
        return (None if op == "COUNT" else out), cnt
    # ---- vectorised
    if n == 0:
        return (None if op == "COUNT" else np.zeros(0, np.int64)), np.zeros(0, np.int64)
    empty = hi < lo
    a_, b_ = np.clip(lo, 0, n), np.clip(np.maximum(hi + 1, lo), 0, n)  # prefix indices; any in range when empty
    cs = np.concatenate([np.zeros(1, np.int64), np.cumsum(ok.astype(np.int64))])
    cnt = np.where(empty, 0, cs[b_] - cs[a_])
    if op == "COUNT":
        return None, cnt
    if op == "SUM_I64":
        u = np.concatenate([np.zeros(1, np.uint64), np.cumsum(np.where(ok, v, 0).view(np.uint64), dtype=np.uint64)])
        out = (u[b_] - u[a_]).view(np.int64)
    elif start is None:  # a run from the segment start, read at hi
        r, _ = segmented_scan(v, ok, offsets, op)
        out = r[np.clip(hi, 0, max(n - 1, 0))] if n else r
    elif end is None:  # a run from the segment end backwards, read at lo
        off = np.asarray(offsets, dtype=np.int64)
        r, _ = segmented_scan(v[::-1].copy(), ok[::-1].copy(), (n - off)[::-1].copy(), op)
        out = r[::-1][np.clip(lo, 0, max(n - 1, 0))] if n else r
    else:  # bounded: windows [i + start, i + end] of a padded copy, masked to [lo, hi] and the valid rows
        s0 = min(max(int(start), -n - 1), n + 1)  # clipped: same frames, no huge windows
        w = min(max(int(end), -n - 1), n + 1) - s0 + 1
        pad = w + abs(s0) + 1
        is_f = op.endswith("F64")
        lo_op = op.startswith("MIN")
        if op == "SUM_F64":
            x, fill = v.view(np.float64), -0.0  # x + -0.0 == x for every x
        else:
            x = _total_order(v) if is_f else v
            fill = np.iinfo(np.int64).max if lo_op else np.iinfo(np.int64).min
        xp = np.concatenate([np.full(pad, fill, dtype=x.dtype), np.where(ok, x, fill), np.full(pad, fill, dtype=x.dtype)])
        out = np.zeros(n, dtype=np.int64)
        step = max(1, 4_000_000 // w)
        for c0 in range(0, n, step):
            c1 = min(n, c0 + step)
            win = np.lib.stride_tricks.sliding_window_view(xp[pad + c0 + s0: pad + c1 + s0 + w - 1], w)
            j = np.arange(c0, c1)[:, None] + s0 + np.arange(w)[None, :]
            win = np.where((j >= lo[c0:c1, None]) & (j <= hi[c0:c1, None]), win, fill)
            if op == "SUM_F64":
                out[c0:c1] = win.sum(axis=1).view(np.int64)
            else:
                red = win.min(axis=1) if lo_op else win.max(axis=1)
                out[c0:c1] = _total_order(red) if is_f else red
    return np.where(cnt > 0, out, 0), cnt


def _frame_column(e: ColumnExpr, st: pa.Table, pdf: Any, offsets: np.ndarray) -> pa.Array:
    """One frame node ``e`` (no alias, no cast) over the sorted table ``st``, in its row order."""
    fn = e.func
    start, end = e.kwargs["rows"]
    n = st.num_rows

    def agg(x: Optional[np.ndarray], ok: Optional[np.ndarray], op: str) -> Tuple[Any, np.ndarray]:
        return frame_aggregate(x, ok, offsets, op, start, end)

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
        return pa.array([(v[j] if ok[j] else None) if k > 0 else None for j, k in zip(r.tolist(), c.tolist())],
                        type=tp)
    if v.dtype == object:
        raise NotImplementedError(f"{fn} on a string column")
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
    """``oracle.window.window_map`` for maps that may hold frame nodes: each distinct frame node becomes a column
    of the input (computed over the same partitions and presort order), the tree reads it, and the rest of the
    map is evaluated by ``oracle.window.window_map``."""
    n = table.num_rows
    sorts = OrderedDict((k, True) for k in keys)
    for k, a in presort.items():  # a key re-listed in the presort takes the presort's direction, as map_dataframe
        sorts[k] = a
    order = S.argsort(table, sorts, "last")
    st = table.take(pa.array(order, type=pa.int64()))
    offsets = np.concatenate([np.flatnonzero(S.group_heads(st, keys)), [n]]).astype(np.int64)
    pdf = W._pandas(st)
    inverse = np.empty(n, dtype=np.int64)
    inverse[order] = np.arange(n)
    temps: Dict[str, pa.Array] = {}

    def replace(e: Any) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if e.kind == Kind.WINDOW and "rows" in e.kwargs:
            bare = e.alias("").cast(None)
            uid = "__f" + bare.fingerprint()[:12]
            if uid not in temps:
                temps[uid] = _frame_column(bare, st, pdf, offsets).take(pa.array(inverse, type=pa.int64()))
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
    return W.window_map(full, keys, presort, exprs)
