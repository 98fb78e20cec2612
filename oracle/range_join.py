"""Oracle: range join reference (``B200ExecutionEngine.range_join``), CPU only.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The rule: left row i and right row j are a pair when their keys are equal (a NULL or NaN key never matches, -0.0
equals 0.0, strings compare by value) and ``start_j <= at_i <= end_j``, each ``<=`` strict where ``closed`` leaves
that side open ("both": neither strict, "left": the upper one, "right": the lower one, "neither": both).  A NULL or
NaN ``at``, ``start`` or ``end`` is never in a pair.  Values compare as their unsigned order codes: a signed or
temporal value v is v + 2^63, an unsigned one itself, a float the usual total-order transform of its bits with
-0.0 read as 0.0; so comparisons are exact over the whole int64 / uint64 range.

Output order: left rows in input order; each row's pairs in ascending (start, right row); ``inner`` drops a left
row without pairs, ``left_outer`` keeps it once with right row -1.

Two levels:

* ``match_pairs`` is the rule written out in plain Python over Python ints, one left row at a time.
* ``match_pairs_np`` has the same contract for one int64 surrogate key and uint64 code arrays: per key group the
  left rows are sorted once and every interval takes its contiguous slice of them, so its cost is the number of
  pairs, not the number of candidates.

``range_join`` applies ``match_pairs`` to Arrow tables and assembles the engine's output table.
"""
import math
import struct
from collections import defaultdict
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

CLOSED = ("both", "left", "right", "neither")
HOWS = ("inner", "left_outer")
_SIGN = 1 << 63


def _sides(closed: str) -> Tuple[bool, bool]:
    assert closed in CLOSED
    return closed in ("both", "left"), closed in ("both", "right")


def holds(start: int, x: int, end: int, closed: str = "both") -> bool:
    """Whether the interval [start, end] (sides by ``closed``) holds x; all three order codes."""
    lo, hi = _sides(closed)
    return (start <= x if lo else start < x) and (x <= end if hi else x < end)


def match_pairs(left_keys: Sequence[Optional[tuple]], left_codes: Sequence[Optional[int]],
                right_keys: Sequence[Optional[tuple]], start_codes: Sequence[Optional[int]],
                end_codes: Sequence[Optional[int]], closed: str = "both", how: str = "inner") -> List[Tuple[int, int]]:
    """The (left row, right row) pairs in output order.  Keys are tuples (None: never matches) and values order
    codes (None: NULL), both already normalised by ``key_tuples`` / ``order_codes``."""
    assert how in HOWS
    runs: Dict[tuple, List[int]] = defaultdict(list)
    for j, k in enumerate(right_keys):
        if k is not None:
            runs[k].append(j)
    out: List[Tuple[int, int]] = []
    for i, (k, x) in enumerate(zip(left_keys, left_codes)):
        hits = []
        if k is not None and x is not None:
            for j in runs.get(k, []):
                s, e = start_codes[j], end_codes[j]
                if s is not None and e is not None and holds(s, x, e, closed):
                    hits.append(j)
        hits.sort(key=lambda j: (start_codes[j], j))
        out.extend((i, j) for j in hits)
        if not hits and how == "left_outer":
            out.append((i, -1))
    return out


def _float_code(v: float) -> int:
    b = struct.unpack("<Q", struct.pack("<d", 0.0 if v == 0 else v))[0]
    return b ^ ((1 << 64) - 1) if b >> 63 else b | _SIGN


def order_codes(arr: Any) -> List[Optional[int]]:
    """An Arrow value column as unsigned order codes (Python ints), None for NULL and NaN."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    tp = arr.type
    if pa.types.is_date32(tp):
        arr = arr.view(pa.int32())
    elif pa.types.is_date64(tp) or pa.types.is_timestamp(tp) or pa.types.is_duration(tp) or pa.types.is_time64(tp):
        arr = arr.view(pa.int64())
    out: List[Optional[int]] = []
    for v in arr.to_pylist():
        if v is None:
            out.append(None)
        elif pa.types.is_floating(tp):
            v = float(v)
            out.append(None if math.isnan(v) else _float_code(v))
        elif pa.types.is_unsigned_integer(tp):
            out.append(int(v))
        else:
            out.append(int(v) + _SIGN)
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


def range_join(left: pa.Table, right: pa.Table, on: Sequence[str], at: str, start: str, end: str,
               how: str = "inner", closed: str = "both") -> pa.Table:
    """The engine's output: for every pair, left's row, then right's columns other than ``on`` (``start`` and
    ``end`` included) from the paired row (NULL for -1)."""
    pairs = match_pairs(key_tuples(left, on), order_codes(left.column(at)), key_tuples(right, on),
                        order_codes(right.column(start)), order_codes(right.column(end)), closed, how)
    out = left.take(pa.array([i for i, _ in pairs], type=pa.int64()))
    idx = pa.array([j if j >= 0 else None for _, j in pairs], type=pa.int64())
    for n in right.column_names:
        if n not in on:
            out = out.append_column(right.schema.field(n), right.column(n).take(idx))
    return out


def codes_np(values: np.ndarray) -> np.ndarray:
    """``order_codes`` of a numpy int64 / uint64 / float64 array as uint64 (NaN rows: meaningless, mask them)."""
    if values.dtype.kind == "f":
        b = np.where(values == 0, 0.0, values).astype(np.float64).view(np.uint64)
        return np.where(b >> np.uint64(63), ~b, b | np.uint64(_SIGN))
    if values.dtype.kind == "u":
        return values.astype(np.uint64)
    return values.astype(np.int64).view(np.uint64) ^ np.uint64(_SIGN)


def match_pairs_np(left_key: np.ndarray, left_code: np.ndarray, left_ok: np.ndarray, right_key: np.ndarray,
                   start_code: np.ndarray, end_code: np.ndarray, right_ok: np.ndarray, closed: str = "both",
                   how: str = "inner") -> Tuple[np.ndarray, np.ndarray]:
    """``match_pairs`` for one int64 key and uint64 codes (``*_ok``: False for a NULL key or value), as two int64
    arrays (left rows, right rows)."""
    assert how in HOWS
    lo_closed, hi_closed = _sides(closed)
    rsel = np.flatnonzero(right_ok & (start_code <= end_code))
    lsel = np.flatnonzero(left_ok)
    lord = lsel[np.lexsort((left_code[lsel], left_key[lsel]))]
    lk, lx = left_key[lord], left_code[lord]
    rord = rsel[np.argsort(right_key[rsel], kind="stable")]
    rk = right_key[rord]
    li_parts, ri_parts = [], []
    bounds = np.flatnonzero(np.diff(rk)) + 1
    for grp in np.split(np.arange(len(rord)), bounds):
        if len(grp) == 0:
            continue
        rj = rord[grp]
        a0, b0 = np.searchsorted(lk, rk[grp[0]], "left"), np.searchsorted(lk, rk[grp[0]], "right")
        xs = lx[a0:b0]
        a = np.searchsorted(xs, start_code[rj], "left" if lo_closed else "right")
        b = np.searchsorted(xs, end_code[rj], "right" if hi_closed else "left")
        cnt = np.maximum(b - a, 0)
        tot = int(cnt.sum())
        if tot == 0:
            continue
        first = np.repeat(a - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt) + np.arange(tot)
        li_parts.append(lord[a0 + first])
        ri_parts.append(np.repeat(rj, cnt))
    li = np.concatenate(li_parts) if li_parts else np.zeros(0, np.int64)
    ri = np.concatenate(ri_parts) if ri_parts else np.zeros(0, np.int64)
    if how == "left_outer":
        lone = np.setdiff1d(np.arange(len(left_key)), li)
        li = np.concatenate([li, lone])
        ri = np.concatenate([ri, np.full(len(lone), -1, np.int64)])
    sc = np.zeros(len(ri), np.uint64)
    sc[ri >= 0] = start_code[ri[ri >= 0]]
    order = np.lexsort((ri, sc, li))
    return li[order].astype(np.int64), ri[order].astype(np.int64)
