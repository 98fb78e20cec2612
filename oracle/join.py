"""Oracle: exact equi-join reference for the K7 hash join (CPU only, numpy / plain Python).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Two levels:

* ``join_pairs`` has the contract of the kernels (``kernels.JoinTable.probe``): keys are 64-bit patterns, every
  pattern is an ordinary key (``0``, ``-1``, ``INT64_MIN``, ``INT64_MAX`` included) and a row whose validity is 0
  never matches.  Built from a stable argsort, ``searchsorted`` and ``repeat``: no per-row Python loop, so it
  joins millions of rows in seconds.
* ``join_rows`` has the contract of ``ExecutionEngine.join`` on Arrow tables, for every join type: NULL keys never
  match, a NaN key never matches (the reference engine works on pandas, where NaN is NULL, and drops such keys
  before it merges: ``native_engine.join``), ``-0.0`` equals ``0.0``, strings compare by value, and right / full
  outer joins take the key from the right row when the left row is missing.  It works on Python values, so unlike
  ``native_engine.join`` (pandas turns a nullable int64 into float64) it is exact near 2^63.
"""
import math
import struct
from collections import Counter
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

JOIN_TYPES = ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti", "cross"]


def _valid(v: Optional[np.ndarray], n: int) -> np.ndarray:
    return np.ones(n, dtype=bool) if v is None else np.asarray(v).astype(bool)


def join_pairs(probe_keys: np.ndarray, probe_valid: Optional[np.ndarray], build_keys: np.ndarray,
               build_valid: Optional[np.ndarray], outer: bool) -> Tuple[np.ndarray, np.ndarray]:
    """(probe_row, build_row) of every match, sorted by probe row, then build row.  With ``outer`` a probe
    row without a match yields ``(i, -1)``."""
    pk = np.ascontiguousarray(probe_keys).view(np.int64)
    bk = np.ascontiguousarray(build_keys).view(np.int64)
    pv, bv = _valid(probe_valid, len(pk)), _valid(build_valid, len(bk))
    brows = np.flatnonzero(bv)
    order = np.argsort(bk[brows], kind="stable")     # equal keys stay in build-row order
    skeys, srows = bk[brows][order], brows[order]
    lo = np.searchsorted(skeys, pk, side="left")
    hi = np.searchsorted(skeys, pk, side="right")
    cnt = np.where(pv, hi - lo, 0).astype(np.int64)
    out_cnt = np.maximum(cnt, 1) if outer else cnt
    total = int(out_cnt.sum())
    probe = np.repeat(np.arange(len(pk), dtype=np.int64), out_cnt)
    start = np.cumsum(out_cnt) - out_cnt
    within = np.arange(total, dtype=np.int64) - np.repeat(start, out_cnt)
    matched = np.repeat(cnt, out_cnt) > 0
    pos = np.repeat(lo, out_cnt) + within
    build = np.full(total, -1, dtype=np.int64)
    build[matched] = srows[pos[matched]]
    return probe, build


def probe_counts(probe_keys: np.ndarray, probe_valid: Optional[np.ndarray], build_keys: np.ndarray,
                 build_valid: Optional[np.ndarray], outer: bool) -> np.ndarray:
    """Output rows per probe row (``JoinTable.probe_counts``)."""
    probe, _ = join_pairs(probe_keys, probe_valid, build_keys, build_valid, outer)
    return np.bincount(probe, minlength=len(probe_keys)).astype(np.int64)


def matched_build_rows(probe_keys: np.ndarray, probe_valid: Optional[np.ndarray], build_keys: np.ndarray,
                       build_valid: Optional[np.ndarray]) -> np.ndarray:
    """1 for every build row that some probe row matches, else 0 (``JoinTable.matched_mask``)."""
    _, build = join_pairs(probe_keys, probe_valid, build_keys, build_valid, False)
    m = np.zeros(len(build_keys), dtype=np.uint8)
    m[build] = 1
    return m


# ---- engine level --------------------------------------------------------------------------------------
def canon(v: Any) -> Any:
    """A value as it is compared in an output row: floats by bit pattern (so ``-0.0`` differs from ``0.0`` and a
    NaN equals the NaN with the same bits), everything else as it is."""
    if isinstance(v, float):
        return ("f64", struct.unpack("<q", struct.pack("<d", v))[0])
    return v


def _join_key(row: dict, on: Sequence[str]) -> Optional[tuple]:
    """The key tuple rows match on, or None when the row matches nothing (a NULL or NaN in any key column)."""
    key = []
    for k in on:
        v = row[k]
        if v is None or (isinstance(v, float) and math.isnan(v)):
            return None
        key.append(0.0 if isinstance(v, float) and v == 0 else v)
    return tuple(key)


def output_names(left: pa.Table, right: pa.Table, how: str, on: Sequence[str]) -> List[str]:
    """Columns of the output: the left table's, then the right table's that are not keys (none for semi / anti)."""
    if how in ("semi", "left_semi", "anti", "left_anti"):
        return list(left.column_names)
    return list(left.column_names) + [c for c in right.column_names if c not in on]


def join_rows(left: pa.Table, right: pa.Table, how: str, on: Sequence[str]) -> Counter:
    """The output of ``left JOIN right`` as a multiset of row tuples (values through ``canon``), columns in the
    order of ``output_names``."""
    how = how.lower()
    if how not in JOIN_TYPES + ["left_semi", "left_anti"]:
        raise ValueError(how)
    on = list(on)
    lrows, rrows = left.to_pylist(), right.to_pylist()
    lnames, rnames = list(left.column_names), [c for c in right.column_names if c not in on]
    out: Counter = Counter()

    def emit(lr: Optional[dict], rr: Optional[dict], semi: bool = False) -> None:
        vals = [None if lr is None else lr[c] for c in lnames]
        if lr is None:  # the key columns of a right row without a left row come from the right row
            vals = [rr[c] if c in on else None for c in lnames]
        if not semi:
            vals += [None if rr is None else rr[c] for c in rnames]
        out[tuple(canon(v) for v in vals)] += 1

    if how == "cross":
        for lr in lrows:
            for rr in rrows:
                emit(lr, rr)
        return out
    index: dict = {}
    for j, rr in enumerate(rrows):
        k = _join_key(rr, on)
        if k is not None:
            index.setdefault(k, []).append(j)
    matched = np.zeros(len(rrows), dtype=bool)
    for lr in lrows:
        k = _join_key(lr, on)
        hits = index.get(k, []) if k is not None else []
        if how in ("semi", "left_semi", "anti", "left_anti"):
            if bool(hits) == (how in ("semi", "left_semi")):
                emit(lr, None, semi=True)
            continue
        for j in hits:
            matched[j] = True
            emit(lr, rrows[j])
        if not hits and how in ("left_outer", "full_outer"):
            emit(lr, None)
    if how in ("right_outer", "full_outer"):
        for j in np.flatnonzero(~matched):
            emit(None, rrows[j])
    return out


def rows_of(table: pa.Table) -> Counter:
    """An engine's output table as the same multiset ``join_rows`` returns."""
    return Counter(tuple(canon(v) for v in r.values()) for r in table.to_pylist())
