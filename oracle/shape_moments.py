"""Exact reference for SKEWNESS / SKEWNESS_POP / KURTOSIS / KURTOSIS_POP.

The central sums Mk = sum of (x - mean)^k (k = 2, 3, 4) over the m non-NULL values are taken exactly over
``fractions.Fraction`` of the float64 values (every finite double is a dyadic rational, and so is their mean times m).
The results need a square root (skewness) and divisions; they are finished in ``decimal`` at 60 significant digits
and rounded to float64 once.  With that many digits the rounding to float64 is correct except when the exact value
lies within 10^-50 relative of a float64 rounding boundary.

    SKEWNESS      G1 = m sqrt(m - 1) / (m - 2) * M3 / M2^1.5                                  NULL when m < 3
    SKEWNESS_POP  g1 = sqrt(m) * M3 / M2^1.5                                                  NULL when m = 0
    KURTOSIS      G2 = m (m + 1)(m - 1) M4 / ((m - 2)(m - 3) M2^2) - 3 (m - 1)^2 / ((m - 2)(m - 3))  NULL when m < 4
    KURTOSIS_POP  g2 = m M4 / M2^2 - 3                                                        NULL when m = 0

M2 = 0 (every value equal) gives 0; a NaN or +-inf among the values gives NaN.  This is exact mathematics, not
pandas: pandas zeroes central sums it takes for rounding noise (below (eps max|x|)^k m) before it divides, so the two
agree only where that does not bite.
"""
import decimal
import math
from fractions import Fraction
from typing import Any, Dict, List, Optional, Sequence, Tuple

FUNCS = ("SKEWNESS", "SKEWNESS_POP", "KURTOSIS", "KURTOSIS_POP")
_MIN_COUNT = {"SKEWNESS": 3, "SKEWNESS_POP": 1, "KURTOSIS": 4, "KURTOSIS_POP": 1}
_CTX = decimal.Context(prec=60)

# (m, M2, M3, M4) of a list of values: M* are Fractions, or None for a non-finite value among them
Moments = Tuple[int, Optional[Fraction], Optional[Fraction], Optional[Fraction]]


def central_sums(values: Sequence[Optional[float]]) -> Moments:
    """(m, M2, M3, M4) of the non-None values, exact; M* are None when m = 0 or a value is not finite."""
    vals = [float(x) for x in values if x is not None]
    m = len(vals)
    if m == 0 or not all(math.isfinite(x) for x in vals):
        return m, None, None, None
    fs = [Fraction(x) for x in vals]
    mean = sum(fs) / m
    ds = [f - mean for f in fs]
    return m, sum(d * d for d in ds), sum(d * d * d for d in ds), sum((d * d) * (d * d) for d in ds)


def _dec(q: Fraction) -> decimal.Decimal:
    return _CTX.divide(decimal.Decimal(q.numerator), decimal.Decimal(q.denominator))


def finish(fn: str, mom: Moments) -> Optional[float]:
    """``fn`` from exact (m, M2, M3, M4): None for NULL, NaN for a non-finite input, else one rounding to float64."""
    assert fn in FUNCS, fn
    m, m2, m3, m4 = mom
    if m < _MIN_COUNT[fn]:
        return None
    if m2 is None:
        return math.nan
    if m2 == 0:
        return 0.0
    if fn.startswith("SKEWNESS"):
        w = Fraction(m * m * (m - 1), (m - 2) ** 2) if fn == "SKEWNESS" else Fraction(m)
        # w^(1/2) * M3 / M2^(3/2) = sign(M3) * sqrt(w * M3^2 / M2^3)
        r = _CTX.sqrt(_dec(w * m3 * m3 / (m2 ** 3)))
        return float(-r if m3 < 0 else r)
    if fn == "KURTOSIS":
        q = Fraction(m * (m + 1) * (m - 1), (m - 2) * (m - 3)) * m4 / (m2 * m2) - \
            Fraction(3 * (m - 1) ** 2, (m - 2) * (m - 3))
    else:
        q = m * m4 / (m2 * m2) - 3
    return float(_dec(q))


def result(fn: str, values: Sequence[Optional[float]]) -> Optional[float]:
    """``fn`` of the non-None values (None: NULL)."""
    return finish(fn, central_sums(values))


def group_results(fn: str, keys: Sequence[Any], values: Sequence[Optional[float]]) -> Dict[Any, Optional[float]]:
    """Per distinct key (None is a key of its own): ``fn`` of its rows' values."""
    groups: Dict[Any, List[Optional[float]]] = {}
    for k, v in zip(keys, values):
        groups.setdefault(k, []).append(v)
    return {k: result(fn, vs) for k, vs in groups.items()}


def running_results(fn: str, values: Sequence[Optional[float]]) -> List[Optional[float]]:
    """Per row, ``fn`` of the non-None values up to and including it (the running window form)."""
    out: List[Optional[float]] = []
    for i in range(len(values)):
        out.append(result(fn, values[:i + 1]))
    return out


def partition_results(fn: str, values: Sequence[Optional[float]]) -> List[Optional[float]]:
    """Per row, ``fn`` over every value of its partition (the whole-partition window form)."""
    r = result(fn, values)
    return [r] * len(values)


def naive_power_sums(fn: str, values: Sequence[float]) -> Optional[float]:
    """``fn`` in float64 from the textbook power sums S1..S4 (M3 = S3 - 3 S1 S2 / m + 2 S1^3 / m^2, ...): the
    formula this engine does not use, kept to show how it fails on data with a large mean."""
    xs = [float(x) for x in values]
    m = len(xs)
    if m < _MIN_COUNT[fn]:
        return None
    s1, s2, s3, s4 = (math.fsum(x ** k for x in xs) for k in (1, 2, 3, 4))
    mu = s1 / m
    m2 = s2 - s1 * mu
    m3 = s3 - 3 * mu * s2 + 2 * m * mu ** 3
    m4 = s4 - 4 * mu * s3 + 6 * mu * mu * s2 - 3 * m * mu ** 4
    if m2 <= 0:
        return 0.0
    if fn == "SKEWNESS":
        return m * math.sqrt(m - 1) / (m - 2) * m3 / m2 ** 1.5
    if fn == "SKEWNESS_POP":
        return math.sqrt(m) * m3 / m2 ** 1.5
    g = m * m4 / (m2 * m2)
    if fn == "KURTOSIS":
        return ((m + 1) * (m - 1) * g - 3 * (m - 1) ** 2) / ((m - 2) * (m - 3))
    return g - 3


U = 2.0 ** -53


def sums_bound(values: Sequence[float], route: str) -> Tuple[float, float, float]:
    """Bounds on |M2 - exact|, |M3 - exact|, |M4 - exact| of finite values for the engine's two algorithms (DESIGN
    §7m), with m values, X = max |x|, D_i = |x_i - mean| and B_k(s) = sum of (D_i + s)^k:

    * ``"hash"``, K6's sums of d^k about the atomically summed mean c (|c - mean| <= e = 2 m u X), corrected on the
      host: (k + 1)(m + 4) u B_k(e).  The rounding of each d_i and of its power and the atomic sum add at most
      (m + 5) u B_k, and the error of delta = DEV / m (u B_1) enters the correction of Mk through k delta D_(k-1),
      at most k m u B_k (Chebyshev's sum inequality B_1 B_(k-1) <= m B_k).
    * ``"scan"``, K9's pairwise updates: 4 (m + 4) u (B_k + k X B_(k-1)); the second term is the error of the running
      means entering the cross terms, as in the variance scan's bound m u ||x|| sqrt(M2).
    """
    xs = [float(x) for x in values]
    m = len(xs)
    mean = float(sum(Fraction(x) for x in xs) / m)
    X = max(abs(x) for x in xs)
    ds = [abs(x - mean) for x in xs]

    def b(k: int, s: float = 0.0) -> float:
        return math.fsum((d + s) ** k for d in ds)

    if route == "hash":
        e = 2 * m * U * X
        return tuple((k + 1) * (m + 4) * U * b(k, e) * 1.01 for k in (2, 3, 4))  # type: ignore[return-value]
    assert route == "scan", route
    return scan_bound(m, X, [b(k) for k in (1, 2, 3, 4)])


def scan_bound(m: Any, X: Any, b: Sequence[Any]) -> Tuple[Any, Any, Any]:
    """The ``"scan"`` bounds of ``sums_bound`` from m, X and b = (B_1, B_2, B_3, B_4); any upper bounds on X and the
    B_k give sound (looser) bounds.  Plain arithmetic, so numpy arrays of rows work as well as floats."""
    return tuple(4 * (m + 4) * U * (b[k - 1] + k * X * b[k - 2]) * 1.01 for k in (2, 3, 4))  # type: ignore


def result_bound(fn: str, values: Sequence[float], route: str) -> float:
    """A bound on |result - exact result| of finite values (m at least the function's minimum count): the
    statistic over the box of central sums within ``sums_bound``, plus eight roundings of the finishing formula.
    Infinite when the box reaches M2 <= 0 (the data is too close to constant for the algorithm to say)."""
    m, *exact = central_sums(values)
    return box_bound(fn, m, [float(q) for q in exact], sums_bound(values, route))


def box_bound(fn: str, m: int, exact: Sequence[float], bounds: Sequence[float]) -> float:
    """``result_bound`` from m, the exact (M2, M3, M4) rounded to float and the bounds on them."""
    e2, e3, e4 = exact
    d2, d3, d4 = bounds
    if e2 == 0 and d2 == 0:
        return 0.0
    if e2 - d2 <= 0:
        return math.inf

    def stat(q2: float, q3: float, q4: float) -> float:
        if fn == "SKEWNESS":
            return m * math.sqrt(m - 1) / (m - 2) * q3 / q2 ** 1.5
        if fn == "SKEWNESS_POP":
            return math.sqrt(m) * q3 / q2 ** 1.5
        g = m * q4 / (q2 * q2)
        if fn == "KURTOSIS":
            return ((m + 1) * (m - 1) * g - 3 * (m - 1) ** 2) / ((m - 2) * (m - 3))
        return g - 3

    c = stat(e2, e3, e4)
    corners = [stat(q2, q3, q4) for q2 in (e2 - d2, e2 + d2) for q3 in (e3 - d3, e3 + d3) for q4 in (e4 - d4, e4 + d4)]
    scale = abs(c) + (3.0 * (m - 1) ** 2 / ((m - 2) * (m - 3)) if fn == "KURTOSIS" else 3.0)
    return max(abs(x - c) for x in corners) + 8 * U * scale
