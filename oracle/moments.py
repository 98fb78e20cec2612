"""Exact reference for VAR_SAMP / VAR_POP / STDDEV_SAMP / STDDEV_POP.

M2 = sum of (x - mean)^2 over the m non-NULL values equals sum(x^2) - sum(x)^2 / m.  Both sums are taken exactly
over ``fractions.Fraction`` of the float64 values (every finite double is a dyadic rational), so M2 is exact and
is rounded to float64 once.  A NaN or +-inf among the values makes M2 NaN.  The results are then:

    VAR_SAMP = M2 / (m - 1)   NULL when m < 2        STDDEV_SAMP = sqrt(VAR_SAMP)
    VAR_POP  = M2 / m         NULL when m = 0        STDDEV_POP  = sqrt(VAR_POP)

each computed from the exact M2 and rounded once (the square root of a correctly rounded quotient for STDDEV:
within 1 ulp of the exact root).
"""
import math
from fractions import Fraction
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

FUNCS = ("VAR_SAMP", "VAR_POP", "STDDEV_SAMP", "STDDEV_POP")


def moments(values: Sequence[Optional[float]]) -> Tuple[int, Optional[float]]:
    """(m, M2 rounded once) of the non-None values; M2 is None when m = 0 and NaN with a non-finite value."""
    vals = [float(x) for x in values if x is not None]
    m = len(vals)
    if m == 0:
        return 0, None
    if not all(math.isfinite(x) for x in vals):
        return m, math.nan
    s = sum(Fraction(x) for x in vals)
    q = sum(Fraction(x) * Fraction(x) for x in vals)
    return m, float(q - s * s / m)


def exact_m2(values: Sequence[float]) -> Fraction:
    """The exact M2 of finite values (no rounding)."""
    s = sum(Fraction(float(x)) for x in values)
    q = sum(Fraction(float(x)) ** 2 for x in values)
    return q - s * s / len(values)


def result(fn: str, m: int, m2: Optional[float]) -> Optional[float]:
    """``fn`` from the count and M2 (None: NULL)."""
    assert fn in FUNCS, fn
    samp = fn.endswith("_SAMP")
    if m < (2 if samp else 1):
        return None
    v = m2 / (m - 1 if samp else m)
    return math.sqrt(v) if fn.startswith("STDDEV") else v


def result_exact(fn: str, values: Sequence[Optional[float]]) -> Optional[float]:
    """``fn`` of the non-None values with ONE rounding of the variance: exact M2 over the exact divisor."""
    vals = [float(x) for x in values if x is not None]
    m = len(vals)
    samp = fn.endswith("_SAMP")
    if m < (2 if samp else 1):
        return None
    if not all(math.isfinite(x) for x in vals):
        return math.nan
    v = float(exact_m2(vals) / (m - 1 if samp else m))
    return math.sqrt(v) if fn.startswith("STDDEV") else v


def group_moments(keys: Sequence[Any], values: Sequence[Optional[float]]) -> Dict[Any, Tuple[int, Optional[float]]]:
    """Per distinct key (None is a key of its own): (m, M2) of its rows' values."""
    groups: Dict[Any, List[Optional[float]]] = {}
    for k, v in zip(keys, values):
        groups.setdefault(k, []).append(v)
    return {k: moments(vs) for k, vs in groups.items()}


def running_moments(values: Sequence[Optional[float]]) -> List[Tuple[int, Optional[float]]]:
    """Per row, (m, M2) of the non-None values up to and including it (exact running sums, one rounding each)."""
    out: List[Tuple[int, Optional[float]]] = []
    s = q = Fraction(0)
    m, bad = 0, False
    for x in values:
        if x is not None:
            x = float(x)
            m += 1
            if not math.isfinite(x):
                bad = True
            else:
                f = Fraction(x)
                s += f
                q += f * f
        out.append((m, None if m == 0 else (math.nan if bad else float(q - s * s / m))))
    return out


def dyadic_group_moments(gid: np.ndarray, k: np.ndarray, valid: Optional[np.ndarray], scale: int = 1024
                         ) -> Dict[int, Tuple[int, Optional[float]]]:
    """(m, M2) per group id of the values k / scale (int64 k, |k| < 2^20, up to 2^22 rows per group: the exact
    integer sums fit in int64), from integer sums instead of fractions: fast enough for millions of rows."""
    gid = np.asarray(gid, dtype=np.int64)
    k = np.asarray(k, dtype=np.int64)
    if valid is not None:
        keep = np.asarray(valid).astype(bool)
        gid, k = gid[keep], k[keep]
    order = np.argsort(gid, kind="stable")
    g, kk = gid[order], k[order]
    starts = np.flatnonzero(np.r_[True, g[1:] != g[:-1]]) if len(g) else np.zeros(0, dtype=np.int64)
    cnt = np.diff(np.r_[starts, len(g)])
    s1 = np.add.reduceat(kk, starts) if len(g) else kk
    s2 = np.add.reduceat(kk * kk, starts) if len(g) else kk
    out: Dict[int, Tuple[int, Optional[float]]] = {}
    for gi, m, a, b in zip(g[starts].tolist(), cnt.tolist(), s1.tolist(), s2.tolist()):
        out[gi] = (m, float(Fraction(b * m - a * a, m * scale * scale)))
    return out
