"""Oracle: the scalar functions of column expressions (CASE, NULLIF, %, ABS, FLOOR, CEIL, ROUND, SQRT, EXP, LN, LOG10,
POWER, GREATEST, LEAST), one Python value at a time.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) - never imported by the product path.

None is NULL.  Integers are Python ints, wrapped to int64 where the engine wraps; floats are Python floats (IEEE
doubles).  ``%`` of integers is the truncated remainder (C, SQL, SQLite, DuckDB; not Python's floor mod); of floats
``math.fmod``, which is exact.  ROUND is exact through ``decimal``.  ``exp`` / ``ln`` / ``log10`` / ``power`` are
computed at 50 digits with ``decimal`` and rounded once to double (``ref_*``): the reference value for the ulp bounds of
the device.  A function that gives NaN for inputs that are not NaN gives NULL (a domain error); a NaN input stays NaN.
``lower`` turns these nodes of expression trees into columns, so that ``oracle/expressions.py`` evaluates the rest.
"""
import decimal
import math
import struct
from typing import Any, List, Optional, Sequence, Tuple

_M64 = (1 << 64) - 1
INT64_MIN = -(1 << 63)
_CTX = decimal.Context(prec=50, Emin=-999999, Emax=999999)


def wrap(v: int) -> int:
    v &= _M64
    return v - (1 << 64) if v >= (1 << 63) else v


def _isnan(v: Any) -> bool:
    return isinstance(v, float) and math.isnan(v)


# ---- per value ----------------------------------------------------------------------------------------------
def mod(a: Any, b: Any, is_float: bool) -> Any:
    if a is None or b is None:
        return None
    if not is_float:
        a, b = int(a), int(b)
        if b == 0:
            return None
        r = abs(a) % abs(b)
        return wrap(-r if a < 0 else r)
    a, b = float(a), float(b)
    if b == 0.0:
        return None
    if _isnan(a) or _isnan(b):
        return math.nan
    if math.isinf(a):
        return None  # fmod(+-inf, y): a domain error
    return math.fmod(a, b)


def abs_(a: Any, is_float: bool) -> Any:
    if a is None:
        return None
    return math.fabs(a) if is_float else wrap(abs(int(a)))


def floor(a: Any, is_float: bool) -> Any:
    if a is None or not is_float:
        return None if a is None else int(a)
    return a if (math.isinf(a) or _isnan(a)) else float(math.floor(a)) if a != 0 else a


def ceil(a: Any, is_float: bool) -> Any:
    if a is None or not is_float:
        return None if a is None else int(a)
    if math.isinf(a) or _isnan(a) or a == 0:
        return a
    r = float(math.ceil(a))
    return -0.0 if r == 0 and a < 0 else r  # ceil(-0.5) is -0.0


def _cround(s: float) -> float:
    """C round: half away from zero, exactly (through decimal)."""
    if math.isinf(s) or _isnan(s) or s == 0:
        return s
    r = float(decimal.Decimal(s).quantize(decimal.Decimal(1), rounding=decimal.ROUND_HALF_UP))
    return math.copysign(r, s) if r == 0 else r


def round_(a: Any, d: int, is_float: bool) -> Any:
    if a is None:
        return None
    if not is_float:
        a = int(a)
        if d >= 0:
            return a
        p = 10 ** -d
        r = abs(a) % p
        q = abs(a) - r + (p if 2 * r >= p else 0)
        return wrap(q if a >= 0 else -q)
    if d == 0:
        return _cround(a)
    p = float(10 ** abs(d))
    s = a * p if d > 0 else a / p
    if math.isinf(s) or _isnan(s):
        return a
    return _cround(s) / p if d > 0 else _cround(s) * p


def sqrt(a: Any) -> Any:
    if a is None:
        return None
    a = float(a)
    if _isnan(a):
        return a
    return None if a < 0 else math.sqrt(a)


def _to_double(x: decimal.Decimal) -> float:
    return float(x)  # the correctly rounded double of the 50-digit value


def ref_exp(a: float) -> float:
    if _isnan(a) or math.isinf(a):
        return a if _isnan(a) or a > 0 else 0.0
    if a > 710.0:  # beyond log(DBL_MAX) = 709.78...: overflows to inf
        return math.inf
    if a < -746.0:  # below log of the smallest subnormal / 2: underflows to 0
        return 0.0
    return _to_double(_CTX.exp(decimal.Decimal(a)))


def ref_ln(a: float) -> Optional[float]:
    if _isnan(a):
        return a
    if a < 0:
        return None
    if a == 0:
        return -math.inf
    if math.isinf(a):
        return a
    return _to_double(_CTX.ln(decimal.Decimal(a)))


def ref_log10(a: float) -> Optional[float]:
    if _isnan(a):
        return a
    if a < 0:
        return None
    if a == 0:
        return -math.inf
    if math.isinf(a):
        return a
    return _to_double(_CTX.log10(decimal.Decimal(a)))


def ref_pow(a: float, b: float) -> Optional[float]:
    """C99 Annex F pow, the finite cases at 50 digits; NaN from non-NaN operands is None."""
    if b == 0 or a == 1.0:
        return 1.0
    if _isnan(a) or _isnan(b):
        return math.nan
    odd_int = math.isfinite(b) and float(b).is_integer() and abs(b) < 2 ** 53 and int(b) % 2 == 1
    if a == 0:  # C99 F.9.4.4; Python's math.pow raises for a negative exponent here
        if b < 0:
            return math.copysign(math.inf, a) if odd_int else math.inf
        return a if odd_int else 0.0
    try:
        r = math.pow(a, b)  # the special cases (infinities, negative bases) as C defines them
    except ValueError:
        return None  # negative finite base, non-integer exponent
    except OverflowError:
        r = None
    if math.isinf(a) or math.isinf(b) or a == 0:
        return r
    try:
        v = _to_double(_CTX.power(decimal.Decimal(abs(a)), decimal.Decimal(b)))
    except decimal.Overflow:
        v = math.inf
    return -v if (a < 0 and odd_int) else v


def total_key(v: float) -> int:
    s = struct.unpack("<q", struct.pack("<d", v))[0]
    return s if s >= 0 else s ^ 0x7FFFFFFFFFFFFFFF


def greatest(vals: Sequence[Any], is_float: bool, least: bool = False) -> Any:
    """NULLs skipped; floats in IEEE totalOrder (bits of the chosen operand kept)."""
    live = [v for v in vals if v is not None]
    if not live:
        return None
    key = (lambda v: total_key(float(v))) if is_float else (lambda v: int(v))
    pick = min(live, key=key) if least else max(live, key=key)
    return float(pick) if is_float else int(pick)


def case(branches: Sequence[Tuple[Any, Any]], else_: Any) -> Any:
    """The value of the first branch whose condition is TRUE (None and False fall through), else ``else_``."""
    for c, v in branches:
        if c is not None and bool(c):
            return v
    return else_


def nullif(a: Any, b: Any) -> Any:
    if a is None:
        return None
    return None if (b is not None and a == b) else a


# ---- expression trees -----------------------------------------------------------------------------------------
_FUNCS = ("CASE", "IF", "IIF", "NULLIF", "IFNULL", "MOD", "ABS", "FLOOR", "CEIL", "CEILING", "ROUND", "SQRT", "EXP",
          "LN", "LOG10", "POWER", "POW", "GREATEST", "LEAST")


def _kind_of(vals: List[Any]) -> str:
    live = [v for v in vals if v is not None]
    if any(isinstance(v, str) for v in live):
        return "s"
    if any(isinstance(v, float) for v in live):
        return "f"
    if live and all(isinstance(v, bool) for v in live):
        return "b"
    return "i"


def lower(df: Any, exprs: List[Any]) -> Tuple[Any, List[Any], List[str]]:
    """Rewrite the scalar-function nodes (and ``%``) of column expressions into named columns holding their values,
    so that ``oracle.expressions`` evaluates the rest.  Returns the pandas frame with the columns added, the rewritten
    expressions (None stays None) and the added names.  A replaced node keeps its alias and cast."""
    import pandas as pd

    from fugue_b200.column import ColumnExpr, Kind, col
    from oracle import expressions as ox

    df = df.copy()
    added: List[str] = []
    n = len(df)

    def values(e: Any) -> Tuple[List[Any], str]:
        v = ox.evaluate(e, df)
        if isinstance(v, pd.Series):
            out = [None if x is pd.NA or (isinstance(x, float) and math.isnan(x)) else x for x in v.tolist()]
            dt = v.dtype
            cls = "f" if pd.api.types.is_float_dtype(dt) else "b" if pd.api.types.is_bool_dtype(dt) else \
                "s" if (pd.api.types.is_string_dtype(dt) or dt == object) else "i"
            return [float(x) if cls == "f" and x is not None else x for x in out], cls
        x = None if v is pd.NA else v
        return [x] * n, ("n" if x is None else _kind_of([x]))

    def unify(classes: List[str]) -> str:
        if "s" in classes:
            return "s"
        return "f" if "f" in classes else ("b" if "b" in classes and all(c in ("b", "n") for c in classes) else "i")

    def conv(v: Any, cls: str) -> Any:
        if v is None:
            return None
        return float(v) if cls == "f" else (bool(v) if cls == "b" else (v if cls == "s" else int(v)))

    def compute(e: ColumnExpr) -> Tuple[List[Any], str]:
        fn = e.head.upper() if e.kind == Kind.CALL else "%"
        args = [a if isinstance(a, ColumnExpr) else ColumnExpr(Kind.LITERAL, a) for a in e.args]
        if fn in ("IF", "IIF"):
            fn, args = "CASE", args
        if fn == "NULLIF":
            (a, ca), (b, _) = values(args[0]), values(args[1])
            return [nullif(x, y) for x, y in zip(a, b)], ca
        if fn in ("CASE",):
            conds = [values(c)[0] for c in args[0:-1:2]]
            res = [values(v) for v in list(args[1:-1:2]) + [args[-1]]]
            cls = unify([c for _, c in res])
            rows = []
            for r in range(n):
                v = case([(conds[j][r], res[j][0][r]) for j in range(len(conds))], res[-1][0][r])
                rows.append(conv(v, cls))
            return rows, cls
        if fn == "IFNULL":
            (a, ca), (b, cb) = values(args[0]), values(args[1])
            cls = unify([ca, cb])
            return [conv(x if x is not None else y, cls) for x, y in zip(a, b)], cls
        if fn in ("%", "MOD"):
            (a, ca), (b, cb) = values(args[0]), values(args[1])
            f = "f" in (ca, cb)
            return [mod(x, y, f) for x, y in zip(a, b)], "f" if f else "i"
        if fn in ("GREATEST", "LEAST"):
            cols = [values(a) for a in args]
            cls = unify([c for _, c in cols])
            rows = [greatest([conv(c[0][r], cls) for c in cols], cls == "f", fn == "LEAST") for r in range(n)]
            return [None if v is None else (bool(v) if cls == "b" else v) for v in rows], cls
        a, ca = values(args[0])
        f = ca == "f"
        if fn == "ABS":
            return [abs_(x, f) for x in a], "f" if f else "i"
        if fn == "FLOOR":
            return [floor(x, f) for x in a], "f" if f else "i"
        if fn in ("CEIL", "CEILING"):
            return [ceil(x, f) for x in a], "f" if f else "i"
        if fn == "ROUND":
            d = args[1].value if len(args) > 1 else 0
            return [round_(x, d, f) for x in a], "f" if f else "i"
        fa = [None if x is None else float(x) for x in a]
        if fn == "SQRT":
            return [sqrt(x) for x in fa], "f"
        if fn in ("EXP", "LN", "LOG10"):
            g = {"EXP": ref_exp, "LN": ref_ln, "LOG10": ref_log10}[fn]
            return [None if x is None else g(x) for x in fa], "f"
        if fn in ("POWER", "POW"):
            b = [None if x is None else float(x) for x in values(args[1])[0]]
            return [None if x is None or y is None else ref_pow(x, y) for x, y in zip(fa, b)], "f"
        raise NotImplementedError(fn)

    def rewrite(e: Any) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if e.has_args:
            e = ColumnExpr(e.kind, e.head, [rewrite(a) for a in e.args], {k: rewrite(v) for k, v in e.kwargs.items()},
                           e.is_distinct, e.as_name, e.as_type)
        if (e.kind == Kind.CALL and e.head.upper() in _FUNCS) or (e.kind == Kind.BINARY and e.head == "%"):
            rows, cls = compute(e)
            name = f"__sc{len(added)}"
            dtype = {"f": "Float64", "b": "boolean", "s": "string", "i": "Int64"}[cls]
            df[name] = pd.array([pd.NA if v is None else v for v in rows], dtype=dtype)
            added.append(name)
            rep = col(name)
            rep = rep.cast(e.as_type) if e.as_type is not None else rep
            return rep.alias(e.as_name) if e.as_name != "" else rep
        return e

    return df, [rewrite(e) for e in exprs], added
