"""Plain-Python reference of NTILE, PERCENT_RANK, CUME_DIST, FIRST_VALUE, LAST_VALUE and NTH_VALUE (DESIGN §4, §7p),
and numpy models of the two kernels that compute them (``fb_window_value``, ``fb_window_distribution``).

The reference takes one row per input row: a partition key (any hashable, None included), one ORDER BY key (int,
float or None; NaN is NULL, -0.0 equals 0.0; ``None`` for the whole list when there is no ORDER BY) and a value, and
returns the head's result per input row.  Rows sort by key in the given direction, NULLs last, ties by input order.
Frames: ``("whole",)``, ``("running",)``, ``("rows", s, e)`` and ``("range", s, e)`` with ``None`` for UNBOUNDED."""
import math
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np


def _norm(k: Any) -> Any:
    if k is None or (isinstance(k, float) and math.isnan(k)):
        return None
    return 0.0 if k == 0 else k


def _partitions(parts: Sequence[Any], keys: Optional[Sequence[Any]], asc: bool) -> List[List[int]]:
    groups: Dict[Any, List[int]] = {}
    for i, p in enumerate(parts):
        groups.setdefault(p, []).append(i)
    out = []
    for rows in groups.values():
        if keys is not None:
            rows = sorted(rows, key=lambda i: (_norm(keys[i]) is None,
                                               0 if _norm(keys[i]) is None else (_norm(keys[i]) if asc else -_norm(keys[i]))))
        out.append(rows)
    return out


def frame_bounds(ks: List[Any], p: int, frame: Tuple[Any, ...], asc: bool) -> Tuple[int, int]:
    """[lo, hi] (positions in the sorted partition; lo > hi: empty) of position p's frame; ``ks`` the sorted keys."""
    n = len(ks)
    kind = frame[0]
    if kind == "whole":
        return 0, n - 1
    if kind == "running":
        return 0, p
    s, e = frame[1], frame[2]
    if kind == "rows":
        return (0 if s is None else max(0, p + s)), (n - 1 if e is None else min(n - 1, p + e))
    k = ks[p]
    if k is None:  # a NULL key's frame is its NULL peers (the partition's tail)
        first_null = next(j for j in range(n) if ks[j] is None)
        return (0 if s is None else first_null), n - 1

    def inside(j: int) -> bool:
        kj = ks[j]
        if kj is None:
            return False
        lo_ok = s is None or (kj >= k + s if asc else kj <= k - s)
        hi_ok = e is None or (kj <= k + e if asc else kj >= k - e)
        return lo_ok and hi_ok

    hits = [j for j in range(n) if inside(j)]
    lo = 0 if s is None else (hits[0] if hits else n)
    hi = n - 1 if e is None else (hits[-1] if hits else -1)
    return lo, hi


def ntile_bucket(r: int, rows: int, n: int) -> int:
    size = rows // n
    if size == 0:
        return r + 1
    large = rows - n * size
    small_from = large * (size + 1)
    return 1 + r // (size + 1) if r < small_from else 1 + large + (r - small_from) // size


def evaluate(head: str, parts: Sequence[Any], keys: Optional[Sequence[Any]], values: Sequence[Any] = (),
             n: Optional[int] = None, frame: Tuple[Any, ...] = ("whole",), asc: bool = True) -> List[Any]:
    out: List[Any] = [None] * len(parts)
    for rows in _partitions(parts, keys, asc):
        ks = [0 if keys is None else _norm(keys[i]) for i in rows]
        N = len(rows)
        for p, i in enumerate(rows):
            if head in ("PERCENT_RANK", "CUME_DIST", "NTILE"):
                pf = min(j for j in range(N) if ks[j] == ks[p])
                pl = max(j for j in range(N) if ks[j] == ks[p])
                if head == "PERCENT_RANK":
                    out[i] = pf / (N - 1) if N > 1 else 0.0
                elif head == "CUME_DIST":
                    out[i] = (pl + 1) / N
                else:
                    out[i] = ntile_bucket(p, N, n)
                continue
            lo, hi = frame_bounds(ks, p, frame, asc)
            j = hi if head == "LAST_VALUE" else lo + (1 if head == "FIRST_VALUE" else n) - 1
            out[i] = values[rows[j]] if lo <= hi and j <= hi else None
    return out


# ---- numpy models of the kernels ---------------------------------------------------------------------------------
TILE = 2048


def rows_frame(i: np.ndarray, sa: np.ndarray, sb: np.ndarray, start: Optional[int], end: Optional[int]
               ) -> Tuple[np.ndarray, np.ndarray]:
    """The ROWS bound helper both frame kernels share: [lo, hi] of rows i in segments [sa, sb)."""
    lo = sa if start is None else np.maximum(sa, i + start)
    hi = sb - 1 if end is None else np.minimum(sb - 1, i + end)
    return lo, hi


def model_value(offsets: np.ndarray, lo: Optional[np.ndarray], hi: Optional[np.ndarray], start: Any, end: Any,
                vals: np.ndarray, valid: np.ndarray, nth: int) -> Tuple[np.ndarray, np.ndarray]:
    """``fb_window_value`` for one column: nth >= 1 or 0 (the frame's last row)."""
    nrows = len(vals)
    i = np.arange(nrows, dtype=np.int64)
    if lo is None:
        seg = np.searchsorted(offsets, i, side="right") - 1
        lo, hi = rows_frame(i, offsets[seg], offsets[seg + 1], start, end)
    else:
        lo, hi = np.maximum(lo, 0), np.minimum(hi, nrows - 1)
    nth = min(nth, nrows + 1)
    j = hi if nth == 0 else lo + nth - 1
    hit = (lo <= hi) & (j <= hi)
    jj = np.where(hit, j, 0)
    ok = hit & (valid[jj] != 0) if nrows else hit
    return np.where(ok, vals[jj] if nrows else vals, 0), ok.astype(np.uint8)


def model_distribution(offsets: np.ndarray, heads: np.ndarray, ntiles: Sequence[int], tile: int = TILE
                       ) -> Tuple[np.ndarray, np.ndarray, List[np.ndarray]]:
    """``fb_window_distribution``: the per-tile first / last head rows, the carry scan over tiles, then every row's
    peer group from its tile and the carries, clipped to its segment."""
    nrows = len(heads)
    ntl = (nrows + tile - 1) // tile
    pos = np.arange(nrows, dtype=np.int64)
    big = np.iinfo(np.int64).max
    tfirst = np.full(ntl, big, np.int64)
    tlast = np.full(ntl, -1, np.int64)
    for t in range(ntl):
        h = pos[t * tile:(t + 1) * tile][heads[t * tile:(t + 1) * tile] != 0]
        if len(h):
            tfirst[t], tlast[t] = h[0], h[-1]
    before = np.concatenate([[-1], np.maximum.accumulate(tlast)[:-1]]) if ntl else tlast
    after = np.concatenate([np.minimum.accumulate(tfirst[::-1])[::-1][1:], [big]]) if ntl else tfirst
    pf = np.empty(nrows, np.int64)
    nx = np.empty(nrows, np.int64)
    for t in range(ntl):
        p, q = before[t], after[t]
        hs = heads[t * tile:(t + 1) * tile]
        for k in range(len(hs)):
            if hs[k]:
                p = t * tile + k
            pf[t * tile + k] = p
        for k in range(len(hs) - 1, -1, -1):
            nx[t * tile + k] = q
            if hs[k]:
                q = t * tile + k
    seg = np.searchsorted(offsets, pos, side="right") - 1
    a, b = offsets[seg], offsets[seg + 1]
    first_peer, last_peer = np.maximum(pf, a), np.minimum(nx, b) - 1
    rows = b - a
    with np.errstate(divide="ignore", invalid="ignore"):
        pr = np.where(rows > 1, (first_peer - a) / np.maximum(rows - 1, 1), 0.0)
        cd = (last_peer - a + 1) / rows
    nts = [np.array([ntile_bucket(int(r), int(m), n) for r, m in zip(pos - a, rows)], np.int64) for n in ntiles]
    return pr, cd, nts
