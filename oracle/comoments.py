"""Exact reference for CORR, COVAR_POP / COVAR_SAMP and the REGR_* aggregates (SQL:2003 binary set functions).

Only the pair rows take part: the m rows where both x and y are non-NULL.  Over them

    Sxx = sum (x - mean x)^2 = sum x^2 - (sum x)^2 / m,   Syy likewise,   Sxy = sum x y - sum x sum y / m

are taken exactly over ``fractions.Fraction`` of the float64 values (every finite double is a dyadic rational), and
every result is computed from the exact sums and rounded to float64 once (a square root within one rounding):

    REGR_COUNT     m (never NULL)                                   COVAR_POP   Sxy / m          NULL when m < 1
    REGR_AVGX / Y  mean of x / y over the pair rows  NULL when m < 1 COVAR_SAMP  Sxy / (m - 1)    NULL when m < 2
    REGR_SXX / SYY / SXY   Sxx / Syy / Sxy                           NULL when m < 1
    REGR_SLOPE     Sxy / Sxx                                        NULL when m < 1 or Sxx = 0
    REGR_INTERCEPT mean y - slope * mean x                          NULL when m < 1 or Sxx = 0
    CORR           Sxy / sqrt(Sxx Syy), in [-1, 1]                  NULL when m < 1 or Sxx = 0 or Syy = 0
    REGR_R2        1 if Syy = 0, else Sxy^2 / (Sxx Syy), in [0, 1]  NULL when m < 1 or Sxx = 0

A NaN or +-inf in x or y of a pair row makes Sxx, Syy and Sxy NaN, so every result built on them is NaN (NaN is
not 0, so the NULL conditions on Sxx and Syy do not hold).  The averages follow AVG: a NaN, or +inf and -inf
together, give NaN, +inf or -inf alone give that infinity.  ``x`` and ``y`` are always passed in that order
here; the SQL argument order (REGR_*(y, x)) is the caller's business.
"""
import math
from fractions import Fraction
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

FUNCS = ("CORR", "COVAR_POP", "COVAR_SAMP", "REGR_COUNT", "REGR_AVGX", "REGR_AVGY", "REGR_SXX", "REGR_SYY",
         "REGR_SXY", "REGR_SLOPE", "REGR_INTERCEPT", "REGR_R2")

# (m, mean x, mean y, Sxx, Syy, Sxy): the exact state, Fractions where finite, float NaN / +-inf otherwise
State = Tuple[int, Any, Any, Any, Any, Any]


def pair_rows(xs: Sequence[Optional[float]], ys: Sequence[Optional[float]]) -> List[Tuple[float, float]]:
    return [(float(x), float(y)) for x, y in zip(xs, ys) if x is not None and y is not None]


def _mean(vals: Sequence[float]) -> Any:
    """AVG of the values: exact for finite ones, else the IEEE sum's NaN / infinity."""
    if any(math.isnan(v) for v in vals) or (math.inf in vals and -math.inf in vals):
        return math.nan
    if math.inf in vals or -math.inf in vals:
        return math.inf if math.inf in vals else -math.inf
    return sum(Fraction(v) for v in vals) / len(vals)


def exact_state(pairs: Sequence[Tuple[float, float]]) -> State:
    m = len(pairs)
    if m == 0:
        return 0, None, None, None, None, None
    xs, ys = [p[0] for p in pairs], [p[1] for p in pairs]
    mx, my = _mean(xs), _mean(ys)
    if not all(math.isfinite(v) for v in xs + ys):
        return m, mx, my, math.nan, math.nan, math.nan
    fx, fy = [Fraction(v) for v in xs], [Fraction(v) for v in ys]
    sx, sy = sum(fx), sum(fy)
    sxx = sum(a * a for a in fx) - sx * sx / m
    syy = sum(b * b for b in fy) - sy * sy / m
    sxy = sum(a * b for a, b in zip(fx, fy)) - sx * sy / m
    return m, mx, my, sxx, syy, sxy


def _sqrt(q: Fraction) -> Fraction:
    """sqrt(q) of a non-negative Fraction to about 80 bits beyond float64 (so one rounding to float64 follows)."""
    if q == 0:
        return Fraction(0)
    k = max(0, (q.denominator.bit_length() - q.numerator.bit_length()) // 2 + 140)
    return Fraction(math.isqrt((q.numerator << (2 * k)) // q.denominator), 1 << k)


def _f(v: Any) -> float:
    return float(v)


def result_of_state(fn: str, st: State) -> Optional[float]:
    """``fn`` of an exact state (None: NULL); the value is rounded once."""
    assert fn in FUNCS, fn
    m, mx, my, sxx, syy, sxy = st
    if fn == "REGR_COUNT":
        return m
    if m < (2 if fn == "COVAR_SAMP" else 1):
        return None
    if fn == "REGR_AVGX":
        return _f(mx)
    if fn == "REGR_AVGY":
        return _f(my)
    nan = isinstance(sxx, float)  # a NaN or an infinity among the pair rows
    if nan:
        return math.nan
    if fn in ("REGR_SXX", "REGR_SYY", "REGR_SXY"):
        return _f({"REGR_SXX": sxx, "REGR_SYY": syy, "REGR_SXY": sxy}[fn])
    if fn in ("COVAR_POP", "COVAR_SAMP"):
        return _f(sxy / (m if fn == "COVAR_POP" else m - 1))
    if sxx == 0:
        return None
    if fn == "REGR_SLOPE":
        return _f(sxy / sxx)
    if fn == "REGR_INTERCEPT":
        return _f(my - sxy / sxx * mx)
    if fn == "REGR_R2":
        return 1.0 if syy == 0 else _f(sxy * sxy / (sxx * syy))
    if syy == 0:  # CORR
        return None
    r = _sqrt(sxy * sxy / (sxx * syy))
    return _f(r if sxy >= 0 else -r)


def result_exact(fn: str, xs: Sequence[Optional[float]], ys: Sequence[Optional[float]]) -> Optional[float]:
    """``fn`` over the pair rows of x and y (rows where either is None are ignored)."""
    return result_of_state(fn, exact_state(pair_rows(xs, ys)))


def group_states(keys: Sequence[Any], xs: Sequence[Optional[float]], ys: Sequence[Optional[float]]
                 ) -> Dict[Any, State]:
    """Per distinct key (None is a key of its own, and a group may have no pair row): its exact state."""
    groups: Dict[Any, List[Tuple[Optional[float], Optional[float]]]] = {}
    for k, x, y in zip(keys, xs, ys):
        groups.setdefault(k, []).append((x, y))
    return {k: exact_state(pair_rows([p[0] for p in v], [p[1] for p in v])) for k, v in groups.items()}


def running_states(xs: Sequence[Optional[float]], ys: Sequence[Optional[float]]) -> List[State]:
    """Per row, the exact state of the pair rows up to and including it (running exact sums)."""
    out: List[State] = []
    sx = sy = sxx = syy = sxy = Fraction(0)
    seen_x: List[float] = []
    seen_y: List[float] = []
    bad = False
    for x, y in zip(xs, ys):
        if x is not None and y is not None:
            x, y = float(x), float(y)
            seen_x.append(x)
            seen_y.append(y)
            if not (math.isfinite(x) and math.isfinite(y)):
                bad = True
            elif not bad:
                a, b = Fraction(x), Fraction(y)
                sx, sy, sxx, syy, sxy = sx + a, sy + b, sxx + a * a, syy + b * b, sxy + a * b
        m = len(seen_x)
        if m == 0:
            out.append((0, None, None, None, None, None))
        elif bad:
            out.append((m, _mean(seen_x), _mean(seen_y), math.nan, math.nan, math.nan))
        else:
            out.append((m, sx / m, sy / m, sxx - sx * sx / m, syy - sy * sy / m, sxy - sx * sy / m))
    return out


def dyadic_group_states(gid: np.ndarray, kx: np.ndarray, ky: np.ndarray, valid: Optional[np.ndarray],
                        scale: int = 1024) -> Dict[int, State]:
    """The exact state per group id of the values kx / scale and ky / scale (int64, |k| < 2^20, up to 2^22 pair rows
    per group, so every integer sum fits in int64), from integer sums: fast enough for millions of rows.
    ``valid`` marks the pair rows (None: all)."""
    gid = np.asarray(gid, dtype=np.int64)
    kx, ky = np.asarray(kx, dtype=np.int64), np.asarray(ky, dtype=np.int64)
    if valid is not None:
        keep = np.asarray(valid).astype(bool)
        gid, kx, ky = gid[keep], kx[keep], ky[keep]
    order = np.argsort(gid, kind="stable")
    g, a, b = gid[order], kx[order], ky[order]
    if len(g) == 0:
        return {}
    starts = np.flatnonzero(np.r_[True, g[1:] != g[:-1]])
    cnt = np.diff(np.r_[starts, len(g)])
    sums = [np.add.reduceat(v, starts) for v in (a, b, a * a, b * b, a * b)]
    out: Dict[int, State] = {}
    s2 = scale * scale
    for gi, m, sa, sb, saa, sbb, sab in zip(g[starts].tolist(), cnt.tolist(), *(s.tolist() for s in sums)):
        out[gi] = (m, Fraction(sa, m * scale), Fraction(sb, m * scale), Fraction(saa * m - sa * sa, m * s2),
                   Fraction(sbb * m - sb * sb, m * s2), Fraction(sab * m - sa * sb, m * s2))
    return out
