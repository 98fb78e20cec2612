"""Oracle: exact CPU reference for PERCENTILE_CONT / PERCENTILE_DISC / MEDIAN (K10), numpy f64 only.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Per group (or segment), the non-NULL values are ordered by ``oracle/sort.null_and_rank`` (a NaN is NULL, -0.0 ties
with 0.0, strings by code point) with ties in row order.  m is their number; m = 0 gives NULL.

* PERCENTILE_CONT(q): the values as float64 (integers rounded to nearest, uint64 as unsigned), then
  ``h = q * (m - 1)``, ``lo = floor(h)``, ``frac = h - lo``; ``x[lo]`` if ``frac == 0`` else
  ``x[lo] + (x[lo + 1] - x[lo]) * frac``, every step one IEEE float64 operation.
* PERCENTILE_DISC(q): the row at sorted position ``max(ceil(q * m) - 1, 0)`` (``q * m`` one float64 multiply).

Groups are keyed by ``oracle/keys.canonical_rows`` (DESIGN §7d).
"""
import math
from typing import Any, Dict, Hashable, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

from .keys import canonical_rows
from .sort import null_and_rank

CONT, DISC = "cont", "disc"


def as_f64(table: pa.Table, name: str) -> np.ndarray:
    """The column as float64 values (NULL rows: 0.0); integers converted by value, rounding to nearest."""
    a = table.column(name).combine_chunks()
    tp = a.type
    if pa.types.is_floating(tp):
        return np.asarray(a.cast(pa.float64()).fill_null(0.0).to_numpy(zero_copy_only=False), dtype=np.float64)
    if pa.types.is_integer(tp):
        return np.array([0.0 if x is None else float(x) for x in a.to_pylist()], dtype=np.float64)
    raise NotImplementedError(f"PERCENTILE_CONT of {tp}")


def sorted_rows(null: np.ndarray, rank: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """The non-NULL rows among ``rows`` in ascending value order, ties in row order."""
    rows = np.asarray(rows, dtype=np.int64)
    keep = rows[~null[rows]]
    return keep[np.lexsort((keep, rank[keep]))]


def cont(x: np.ndarray, q: float) -> Optional[float]:
    """PERCENTILE_CONT of values ``x`` already in sorted order (None when empty)."""
    m = len(x)
    if m == 0:
        return None
    h = np.float64(q) * np.float64(m - 1)
    lo = np.floor(h)
    frac = h - lo
    i = int(lo)
    if frac == 0:
        return float(x[i])
    a, b = np.float64(x[i]), np.float64(x[i + 1])
    with np.errstate(invalid="ignore", over="ignore"):  # inf - inf is NaN, as on the device
        return float(a + (b - a) * frac)


def disc_position(m: int, q: float) -> Optional[int]:
    """Sorted position picked by PERCENTILE_DISC among m values (None when m = 0)."""
    if m == 0:
        return None
    return max(int(math.ceil(float(np.float64(q) * np.float64(m)))) - 1, 0)


def quantiles_of(table: pa.Table, name: str, rows: np.ndarray, qs: Sequence[Tuple[float, str]],
                 null: Optional[np.ndarray] = None, rank: Optional[np.ndarray] = None,
                 x: Optional[np.ndarray] = None) -> Tuple[int, List[Any]]:
    """(m, per q: the CONT float or None, the DISC row index or None) over the rows ``rows`` of column ``name``."""
    if null is None or rank is None:
        null, rank = null_and_rank(table, name)
    order = sorted_rows(null, rank, rows)
    out: List[Any] = []
    for q, kind in qs:
        if kind == CONT:
            if x is None:
                x = as_f64(table, name)
            out.append(cont(x[order], q))
        else:
            p = disc_position(len(order), q)
            out.append(None if p is None else int(order[p]))
    return len(order), out


def segment_quantiles(table: pa.Table, name: str, offsets: np.ndarray,
                      qs: Sequence[Tuple[float, str]]) -> Tuple[np.ndarray, List[List[Any]]]:
    """Per segment ``[offsets[s], offsets[s + 1])``: m, and per q the result list over the segments."""
    null, rank = null_and_rank(table, name)
    x = as_f64(table, name) if any(k == CONT for _, k in qs) else None
    counts, res = [], [[] for _ in qs]
    for s in range(len(offsets) - 1):
        m, r = quantiles_of(table, name, np.arange(offsets[s], offsets[s + 1]), qs, null, rank, x)
        counts.append(m)
        for j, v in enumerate(r):
            res[j].append(v)
    return np.asarray(counts, dtype=np.int64), res


def group_rows(table: pa.Table, keys: Sequence[str]) -> Dict[Hashable, np.ndarray]:
    """Canonical key tuple -> the group's rows in input order (one group of every row without keys)."""
    if not keys:
        return {(): np.arange(table.num_rows, dtype=np.int64)}
    groups: Dict[Hashable, List[int]] = {}
    for i, k in enumerate(canonical_rows(table, keys)):
        groups.setdefault(k, []).append(i)
    return {k: np.asarray(v, dtype=np.int64) for k, v in groups.items()}


def group_quantiles(table: pa.Table, keys: Sequence[str], name: str,
                    qs: Sequence[Tuple[float, str]]) -> Dict[Hashable, Tuple[int, List[Any]]]:
    """Canonical key tuple -> (m, results) of column ``name`` per GROUP BY ``keys`` group."""
    null, rank = null_and_rank(table, name)
    x = as_f64(table, name) if any(k == CONT for _, k in qs) else None
    return {k: quantiles_of(table, name, rows, qs, null, rank, x) for k, rows in group_rows(table, keys).items()}


def window_quantile(table: pa.Table, keys: Sequence[str], name: str, q: float, kind: str) -> List[Any]:
    """Per row, the quantile of its logical partition (keys): the CONT float, or the DISC pick's python value."""
    vals = table.column(name).to_pylist()
    out: List[Any] = [None] * table.num_rows
    null, rank = null_and_rank(table, name)
    x = as_f64(table, name) if kind == CONT else None
    for rows in group_rows(table, keys).values():
        _, (r,) = quantiles_of(table, name, rows, [(q, kind)], null, rank, x)
        v = r if kind == CONT or r is None else vals[r]
        for i in rows:
            out[i] = v
    return out
