"""Oracle: as-of join reference (``B200ExecutionEngine.asof_join``, ``pandas.merge_asof`` semantics), CPU only.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The rule, per left row i: the candidates are the right rows whose key equals i's key and whose as-of value is
not NULL (a NULL or NaN key never matches, -0.0 equals 0.0, strings compare by value; a NULL or NaN as-of value
on the left matches nothing).

* ``backward``: the largest t_r <= t_i (< without ``allow_exact_matches``); among equal t_r the last right row.
* ``forward``: the smallest t_r >= t_i (>); among equal t_r the first right row.
* ``nearest``: the closer of those two; on equal distance the backward one.

A candidate farther than ``tolerance`` is none (no fallback to a farther row).  Integer and temporal distances
are exact (temporal values are their storage integers); a float distance is one f64 subtraction, 0 for equal
values (so +inf is at distance 0 from +inf).

Two levels:

* ``match_rows`` is the rule written out in plain Python over Python values, one left row at a time.
* ``match_rows_np`` has the same contract for one int64 surrogate key and numpy value arrays, with a
  ``searchsorted`` per key group, so it matches millions of rows in seconds.

``asof_join`` applies ``match_rows`` to Arrow tables and assembles the engine's output table.
"""
import math
from collections import defaultdict
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import pyarrow as pa

DIRECTIONS = ("backward", "forward", "nearest")


def _distance(a: Any, b: Any) -> Any:
    return 0 if a == b else abs(a - b)


def match_rows(left_keys: Sequence[Optional[tuple]], left_vals: Sequence[Any], right_keys: Sequence[Optional[tuple]],
               right_vals: Sequence[Any], direction: str = "backward", allow_exact_matches: bool = True,
               tolerance: Any = None) -> List[int]:
    """Per left row the right row it matches, -1 for none.  Keys are tuples (None: never matches) and values
    Python numbers (None: NULL), both already normalised by ``key_tuples`` / ``as_values``."""
    assert direction in DIRECTIONS
    runs: Dict[tuple, List[int]] = defaultdict(list)
    for j, (k, t) in enumerate(zip(right_keys, right_vals)):
        if k is not None and t is not None:
            runs[k].append(j)
    out = []
    for k, x in zip(left_keys, left_vals):
        back = fwd = None
        if k is not None and x is not None:
            for j in runs.get(k, []):
                t = right_vals[j]
                if (t <= x if allow_exact_matches else t < x) and (back is None or t >= right_vals[back]):
                    back = j  # >=: a later row of an equal value replaces the earlier one
                if (t >= x if allow_exact_matches else t > x) and (fwd is None or t < right_vals[fwd]):
                    fwd = j  # <: the first row of an equal value stays
        if tolerance is not None:
            if back is not None and _distance(x, right_vals[back]) > tolerance:
                back = None
            if fwd is not None and _distance(right_vals[fwd], x) > tolerance:
                fwd = None
        if direction == "backward":
            pick = back
        elif direction == "forward":
            pick = fwd
        elif back is None or fwd is None:
            pick = fwd if back is None else back
        else:
            pick = back if _distance(x, right_vals[back]) <= _distance(right_vals[fwd], x) else fwd
        out.append(-1 if pick is None else pick)
    return out


def as_values(arr: Any) -> List[Any]:
    """An Arrow as-of column as Python numbers: temporal types as their storage integers, floats as floats with
    -0.0 read as 0.0, NULL and NaN as None."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    tp = arr.type
    if pa.types.is_date32(tp):
        arr = arr.view(pa.int32())
    elif pa.types.is_date64(tp) or pa.types.is_timestamp(tp) or pa.types.is_duration(tp) or pa.types.is_time64(tp):
        arr = arr.view(pa.int64())
    out = []
    for v in arr.to_pylist():
        if v is not None and pa.types.is_floating(tp):
            v = float(v)
            v = None if math.isnan(v) else (0.0 if v == 0 else v)
        out.append(v)
    return out


def key_tuples(table: pa.Table, on: Sequence[str]) -> List[Optional[tuple]]:
    """Every row's key tuple, None where a key is NULL or NaN (floats: -0.0 equals 0.0 as Python numbers)."""
    cols = [table.column(k).to_pylist() for k in on]
    out: List[Optional[tuple]] = []
    for i in range(table.num_rows):
        vals = tuple(c[i] for c in cols)
        bad = any(v is None or (isinstance(v, float) and math.isnan(v)) for v in vals)
        out.append(None if bad else vals)
    return out


def asof_join(left: pa.Table, right: pa.Table, on: Sequence[str], asof: str, how: str = "inner",
              direction: str = "backward", allow_exact_matches: bool = True, tolerance: Any = None) -> pa.Table:
    """The engine's output: ``left``'s rows in order (only the matched ones for ``inner``), then right's columns
    other than ``on`` and ``asof`` from the matched row (NULL for none).  ``tolerance`` in storage units."""
    m = match_rows(key_tuples(left, on), as_values(left.column(asof)), key_tuples(right, on),
                   as_values(right.column(asof)), direction, allow_exact_matches, tolerance)
    rows = [i for i, j in enumerate(m)] if how == "left_outer" else [i for i, j in enumerate(m) if j >= 0]
    names2 = [n for n in right.column_names if n not in on and n != asof]
    out = left.take(pa.array(rows, type=pa.int64()))
    idx = pa.array([m[i] if m[i] >= 0 else None for i in rows], type=pa.int64())
    for n in names2:
        out = out.append_column(right.schema.field(n), right.column(n).take(idx))
    return out


def _dist_np(lo: np.ndarray, hi: np.ndarray) -> np.ndarray:
    """hi - lo for hi >= lo elementwise: exact (uint64) for integers, f64 (0 where equal) for floats."""
    if lo.dtype.kind == "f":
        return np.where(lo == hi, 0.0, hi - lo)
    sign = np.uint64(1 << 63) if lo.dtype.kind == "i" else np.uint64(0)
    with np.errstate(over="ignore"):
        return (hi.view(np.uint64) ^ sign) - (lo.view(np.uint64) ^ sign)


def match_rows_np(left_key: np.ndarray, left_val: np.ndarray, left_ok: np.ndarray, right_key: np.ndarray,
                  right_val: np.ndarray, right_ok: np.ndarray, direction: str = "backward",
                  allow_exact_matches: bool = True, tolerance: Any = None) -> np.ndarray:
    """``match_rows`` for one int64 key (``*_ok``: bool, False for a NULL key or value) and value arrays of one dtype
    (int64, uint64 or float64 with -0.0 as 0.0)."""
    assert direction in DIRECTIONS and left_val.dtype == right_val.dtype
    out = np.full(len(left_key), -1, dtype=np.int64)
    rsel = np.flatnonzero(right_ok)
    order = np.lexsort((right_val[rsel], right_key[rsel]))  # stable: equal (key, value) keep row order
    rows = rsel[order]
    sk, sv = right_key[rows], right_val[rows]
    lsel = np.flatnonzero(left_ok)
    lord = lsel[np.argsort(left_key[lsel], kind="stable")]
    lk = left_key[lord]
    bounds = np.flatnonzero(np.diff(lk)) + 1
    for grp in np.split(np.arange(len(lord)), bounds):
        if len(grp) == 0:
            continue
        li = lord[grp]
        s, e = np.searchsorted(sk, lk[grp[0]], "left"), np.searchsorted(sk, lk[grp[0]], "right")
        if s == e:
            continue
        run, x = sv[s:e], left_val[li]
        ub, lb = np.searchsorted(run, x, "right"), np.searchsorted(run, x, "left")
        b = (ub if allow_exact_matches else lb) - 1
        f = lb if allow_exact_matches else ub
        hb, hf = b >= 0, f < len(run)
        db = _dist_np(run[np.clip(b, 0, len(run) - 1)], x)
        df = _dist_np(x, run[np.clip(f, 0, len(run) - 1)])
        if tolerance is not None:
            tol = np.float64(tolerance) if run.dtype.kind == "f" else np.uint64(tolerance)
            hb &= db <= tol
            hf &= df <= tol
        if direction == "backward":
            use_b, use_f = hb, np.zeros_like(hf)
        elif direction == "forward":
            use_b, use_f = np.zeros_like(hb), hf
        else:
            use_b = hb & (~hf | (db <= df))
            use_f = hf & ~use_b
        res = np.full(len(li), -1, dtype=np.int64)
        res[use_b] = rows[s + b[use_b]]
        res[use_f] = rows[s + f[use_f]]
        out[li] = res
    return out

