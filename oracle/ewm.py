"""Exact reference of the exponentially weighted mean / var / std of ``fb_segmented_ewm`` (DESIGN §7s), pandas' ``ewm``.

An observation is a value that is neither None nor NaN.  Seen from row i, observation j <= i weighs
w_j beta^(p_last - p_j) with beta = 1 - alpha, p the position (row index, observation ordinal with ``ignore_na``, or
time / halflife with ``times``, beta^dp then 0.5^(dt / halflife)) and p_last the last observation's.  The first
observation has w = 1; with ``adjust`` every other too, else w_k = alpha T_(k-1), T the running total weight.  The sums
run in exact rationals (alpha is a float, so Fraction(alpha) is exact) or, for a time decay, 60-digit decimals, and each
result is rounded once.  A +-inf observation makes the mean +-inf (NaN with both signs) and the variance NaN.
"""
import math
from decimal import Context, Decimal, localcontext
from fractions import Fraction
from typing import Any, List, Optional, Sequence, Tuple

_CTX = Context(prec=60)


def _num(x: Any, decimal: bool) -> Any:
    return _CTX.create_decimal(x) if decimal else Fraction(x)


def _ewm_sums(values: Sequence[Optional[float]], alpha: float, adjust: bool = True, ignore_na: bool = False,
             times: Optional[Sequence[int]] = None, halflife: Any = None,
             decimal: bool = False) -> List[Optional[Tuple[Any, ...]]]:
    """Per row of one partition: None before the first observation, else (count, W, W2, S1, S2, infs) over the
    observations so far (S1 = sum of w x, S2 = sum of w x^2 over the finite ones; infs the set of signs of the
    infinite ones), exact; in 60-digit decimals for a time decay or with ``decimal`` (long partitions, where exact
    rationals grow by the bits of beta at every row)."""
    dec = times is not None or decimal
    beta = _CTX.subtract(_num(1, True), _num(alpha, True)) if dec else 1 - Fraction(alpha)
    a = _num(0.5 if times is not None else alpha, dec)
    one = _num(1, dec)
    out: List[Optional[Tuple[Any, ...]]] = []
    state = None  # (count, W, W2, S1, S2, infs, last position)
    nobs = 0
    for i, x in enumerate(values):
        obs = x is not None and not (isinstance(x, float) and math.isnan(x))
        if not obs:
            out.append(None if state is None else state[:6])
            continue
        nobs += 1
        p = int(times[i]) if times is not None else (nobs - 1 if ignore_na else i)
        if state is None:
            w = one
            c, W, W2, S1, S2, infs = 1, _num(0, dec), _num(0, dec), _num(0, dec), _num(0, dec), frozenset()
        else:
            c, W, W2, S1, S2, infs, last = state
            dp = p - last
            if times is not None:
                d = _CTX.power(_CTX.create_decimal("0.5"), _CTX.divide(_CTX.create_decimal(dp), _num(halflife, True)))
            elif dec:
                d = _CTX.power(beta, dp)
            else:
                d = beta ** dp
            w = one if adjust else a * W
            W, W2, S1, S2 = W * d, W2 * d * d, S1 * d, S2 * d
            c += 1
        W, W2 = W + w, W2 + w * w
        if math.isinf(x):
            infs = infs | {x > 0}
        else:
            xv = _num(x, dec)
            S1, S2 = S1 + w * xv, S2 + w * xv * xv
        state = (c, W, W2, S1, S2, infs, p)
        out.append(state[:6])
    return out


def _f(x: Any) -> float:
    return float(x)


def _ewm_result(fn: str, s: Optional[Tuple[Any, ...]], bias: bool = False, min_periods: int = 0) -> Optional[float]:
    """``fn`` (EWM_MEAN / EWM_VAR / EWM_STD) of one row's sums, rounded once; None for NULL."""
    if s is None:
        return None
    c, W, W2, S1, S2, infs = s
    if c < max(min_periods, 1):
        return None
    if fn != "EWM_MEAN" and not bias and W * W - W2 == 0:
        return None
    if infs:
        if fn != "EWM_MEAN":
            return math.nan
        return math.nan if len(infs) == 2 else (math.inf if True in infs else -math.inf)
    mean = S1 / W
    if fn == "EWM_MEAN":
        return _f(mean)
    var = (S2 - S1 * mean) / W
    if not bias:
        var = var * W * W / (W * W - W2)
    if fn == "EWM_VAR":
        return _f(var)
    v = var if isinstance(var, Decimal) else _CTX.divide(Decimal(var.numerator), Decimal(var.denominator))
    return _f(_CTX.sqrt(v))


def ewm_sums(*args: Any, **kw: Any) -> List[Optional[Tuple[Any, ...]]]:
    """:func:`_ewm_sums`, decimal arithmetic at 60 digits."""
    with localcontext(_CTX):
        return _ewm_sums(*args, **kw)


def ewm_result(*args: Any, **kw: Any) -> Optional[float]:
    """:func:`_ewm_result`, decimal arithmetic at 60 digits."""
    with localcontext(_CTX):
        return _ewm_result(*args, **kw)


def ewm(fn: str, values: Sequence[Optional[float]], alpha: float, adjust: bool = True, ignore_na: bool = False,
        bias: bool = False, min_periods: int = 0, times: Optional[Sequence[int]] = None,
        halflife: Any = None, decimal: bool = False) -> List[Optional[float]]:
    """``fn`` over one partition, row by row."""
    return [ewm_result(fn, s, bias, min_periods)
            for s in ewm_sums(values, alpha, adjust, ignore_na, times, halflife, decimal)]


def pandas_alpha(com: Any = None, span: Any = None, halflife: Any = None, alpha: Any = None) -> float:
    """pandas' alpha of a decay, through the center of mass in float64 as pandas computes it."""
    if com is None:
        com = (span - 1) / 2 if span is not None else (
            1 / (1 - math.exp(math.log(0.5) / halflife)) - 1 if halflife is not None else (1 - alpha) / alpha)
    return 1 / (1 + com)
