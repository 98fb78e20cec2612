"""Oracle: date and timestamp expressions (temporal literals, EXTRACT, DATE_TRUNC, DATEDIFF, ADD_MONTHS, casts between
temporal types, a date / timestamp moved by an interval), one Python value at a time.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) - never imported by the product path.

None is NULL.  A value is a Python int: a count of ``unit`` ("D", "s", "ms", "us", "ns") since 1970-01-01 00:00 UTC.
The calendar is Python's ``datetime.date`` (proleptic Gregorian), reached for any year through the calendar's period of
400 years = 146 097 days = 20 871 weeks: a day count is moved by whole periods into years 401-800, where ``date`` does
the work (year, month, day, ordinal day, ISO week), and the year is moved back.  Every division is Python's floor
division on unbounded ints; results that the engine keeps in int64 are wrapped where it wraps and clamped where it
saturates.  ``lower`` turns these nodes of expression trees into columns, so that ``oracle/expressions.py`` evaluates the
rest; its frames hold temporal columns as their int64 storage values, with the Arrow types given beside them.
"""
import calendar
import datetime
from typing import Any, Dict, List, Optional, Tuple

import pyarrow as pa

PER_DAY = {"D": 1, "s": 86400, "ms": 86400 * 10 ** 3, "us": 86400 * 10 ** 6, "ns": 86400 * 10 ** 9}
FIELDS = ("year", "month", "day", "hour", "minute", "second", "quarter", "dow", "isodow", "doy", "week", "isoyear",
          "epoch")
PARTS = ("year", "quarter", "month", "week", "day", "hour", "minute", "second")
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
_PERIOD = 146097
_ORDINAL_1970 = datetime.date(1970, 1, 1).toordinal()


def wrap(v: int) -> int:
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >= (1 << 63) else v


def clamp(v: int) -> int:
    return min(max(v, INT64_MIN), INT64_MAX)


def unit_of(tp: pa.DataType) -> Optional[str]:
    """The unit of a date / timestamp / duration type; None for any other type."""
    if pa.types.is_date32(tp):
        return "D"
    if pa.types.is_date64(tp):
        return "ms"
    if pa.types.is_timestamp(tp) or pa.types.is_duration(tp):
        return tp.unit
    return None


# ---- calendar ------------------------------------------------------------------------------------------------
def _date_of(days: int) -> Tuple[datetime.date, int]:
    """(the date of ``days`` moved into years 401-800, the years to add back)."""
    q, r = divmod(days + _ORDINAL_1970 - 1, _PERIOD)
    return datetime.date.fromordinal(r + 1 + _PERIOD), (q - 1) * 400


def civil(days: int) -> Tuple[int, int, int]:
    d, dy = _date_of(days)
    return d.year + dy, d.month, d.day


def days_of(y: int, m: int, d: int) -> int:
    q, r = divmod(y - 1, 400)
    return datetime.date(r + 401, m, d).toordinal() + (q - 1) * _PERIOD - _ORDINAL_1970


def split(v: int, unit: str) -> Tuple[int, int]:
    """(days since the epoch, units into that day)."""
    return divmod(v, PER_DAY[unit])


def extract(field: str, v: Optional[int], unit: str) -> Any:
    if v is None:
        return None
    if field == "epoch":  # the engine's rule: one IEEE operation on the stored value converted to a double
        return float(v) * 86400.0 if unit == "D" else float(v) / float(PER_DAY[unit] // 86400)
    days, rem = split(v, unit)
    sod = rem // (PER_DAY[unit] // 86400) if unit != "D" else 0
    d, dy = _date_of(days)
    iso = d.isocalendar()
    return {"year": d.year + dy, "month": d.month, "day": d.day, "hour": sod // 3600, "minute": sod // 60 % 60,
            "second": sod % 60, "quarter": (d.month - 1) // 3 + 1, "dow": iso[2] % 7, "isodow": iso[2],
            "doy": d.timetuple().tm_yday, "week": iso[1], "isoyear": iso[0] + dy}[field]


def date_trunc(part: str, v: Optional[int], unit: str) -> Optional[int]:
    if v is None:
        return None
    per = PER_DAY[unit]
    days, rem = split(v, unit)
    if part in ("hour", "minute", "second"):
        if unit == "D":
            return v
        step = per // 86400 * {"hour": 3600, "minute": 60, "second": 1}[part]
        return wrap(days * per + rem - rem % step)
    if part == "week":
        days -= _date_of(days)[0].isocalendar()[2] - 1
    elif part != "day":
        y, m, _ = civil(days)
        days = days_of(y, 1 if part == "year" else (m - 1) // 3 * 3 + 1 if part == "quarter" else m, 1)
    return wrap(days * per)


def index(part: str, v: int, unit: str) -> int:
    """Whole parts from 1970-01-01 00:00 (weeks: from Monday 1969-12-29) to ``v``."""
    days, rem = split(v, unit)
    sod = rem // (PER_DAY[unit] // 86400) if unit != "D" else 0
    if part in ("hour", "minute", "second"):
        return (days * 86400 + sod) // {"hour": 3600, "minute": 60, "second": 1}[part]
    if part == "day":
        return days
    if part == "week":
        return (days + 3) // 7
    y, m, _ = civil(days)
    return {"year": y - 1970, "quarter": (y - 1970) * 4 + (m - 1) // 3, "month": (y - 1970) * 12 + m - 1}[part]


def datediff(part: str, a: Optional[int], unit_a: str, b: Optional[int], unit_b: str) -> Optional[int]:
    if a is None or b is None:
        return None
    return wrap(index(part, b, unit_b) - index(part, a, unit_a))


def add_months(v: Optional[int], n: Optional[int], unit: str) -> Optional[int]:
    if v is None or n is None:
        return None
    days, rem = split(v, unit)
    y, m, d = civil(days)
    y2, m2 = divmod(y * 12 + m - 1 + n, 12)
    last = calendar.monthrange((y2 - 1) % 400 + 401, m2 + 1)[1]
    return wrap(days_of(y2, m2 + 1, min(d, last)) * PER_DAY[unit] + rem)


def cast(v: Optional[int], unit_from: str, unit_to: str) -> Optional[int]:
    """Coarser -> finer: a saturating multiply; finer -> coarser: a floor division."""
    if v is None:
        return None
    a, b = PER_DAY[unit_from], PER_DAY[unit_to]
    return clamp(v * (b // a)) if b >= a else v // (a // b)


def literal_us(v: Any) -> int:
    """A date / datetime (naive, UTC) / timedelta as exact microseconds (a date is its midnight)."""
    us = datetime.timedelta(microseconds=1)
    if isinstance(v, datetime.timedelta):
        return v // us
    if not isinstance(v, datetime.datetime):
        v = datetime.datetime(v.year, v.month, v.day)
    return (v - datetime.datetime(1970, 1, 1)) // us


def compare(op: str, x: Optional[int], unit: str, literal: Any) -> Optional[bool]:
    """``x op literal`` as mathematics: the stored count against the literal's exact (rational) value in ``unit``."""
    if x is None:
        return None
    lhs, rhs = x * PER_DAY["us"], literal_us(literal) * PER_DAY[unit]  # both in 1 / (us * unit) of a day
    return {"<": lhs < rhs, "<=": lhs <= rhs, ">": lhs > rhs, ">=": lhs >= rhs, "==": lhs == rhs, "!=": lhs != rhs}[op]


def literal_in(v: Any, unit: str) -> int:
    """A literal that is a whole number of ``unit`` as that number (clamped to int64); ValueError otherwise."""
    q, r = divmod(literal_us(v) * PER_DAY[unit], PER_DAY["us"])
    if r:
        raise ValueError(f"{v!r} is not a whole number of {unit}")
    return clamp(q)


# ---- expression trees -----------------------------------------------------------------------------------------
_FUNCS = ("EXTRACT", "DATE_TRUNC", "DATEDIFF", "ADD_MONTHS")
_TEMPORAL = (datetime.date, datetime.datetime, datetime.timedelta)
_NATURAL = {datetime.timedelta: pa.duration("us"), datetime.datetime: pa.timestamp("us"), datetime.date: pa.date32()}
_FLIP = {"<": ">", "<=": ">=", ">": "<", ">=": "<=", "==": "==", "!=": "!="}


def lower(df: Any, exprs: List[Any], types: Dict[str, pa.DataType]) -> Tuple[Any, List[Any], List[str]]:
    """Rewrite the temporal nodes of column expressions into named Int64 / Float64 / boolean columns holding their
    values, so that ``oracle.expressions`` evaluates the rest.  ``df`` holds temporal columns as their int64 storage
    values; ``types`` gives their Arrow types.  Returns the frame with the columns added, the rewritten expressions
    (None stays None) and the added names.  A replaced node keeps its alias, and a cast that is not temporal."""
    import pandas as pd

    from fugue_b200.column import ColumnExpr, Kind, col, lit
    from oracle import expressions as ox

    df = df.copy()
    types = dict(types)
    added: List[str] = []
    n = len(df)

    def is_lit(e: Any) -> bool:
        return isinstance(e, ColumnExpr) and e.kind == Kind.LITERAL and e.as_type is None and isinstance(e.value, _TEMPORAL)

    def ttype(e: Any) -> Optional[pa.DataType]:
        if not isinstance(e, ColumnExpr):
            return None
        if e.as_type is not None:
            return e.as_type if unit_of(e.as_type) else None
        if e.kind == Kind.NAMED:
            return types.get(e.name)
        if is_lit(e):
            return _NATURAL[type(e.value)] if type(e.value) in _NATURAL else pa.timestamp("us")
        if e.kind == Kind.CALL and e.head.upper() in ("DATE_TRUNC", "ADD_MONTHS"):
            return ttype(e.args[0])
        return None

    def values(e: Any) -> List[Any]:
        v = ox.evaluate(e, df)
        if isinstance(v, pd.Series):
            return [None if x is pd.NA else int(x) for x in v.tolist()]
        return [None if v is pd.NA else int(v)] * n

    def column(rows: List[Any], dtype: str, e: Any, tp: Optional[pa.DataType], keep_cast: bool = True) -> Any:
        name = f"__tm{len(added)}"
        df[name] = pd.array([pd.NA if v is None else v for v in rows], dtype=dtype)
        added.append(name)
        if tp is not None:
            types[name] = tp
        rep = col(name)
        if keep_cast and e.as_type is not None and unit_of(e.as_type) is None:
            rep = rep.cast(e.as_type)
        return rep.alias(e.as_name) if e.as_name != "" else rep

    def plain(e: Any) -> Any:
        """A temporal literal alone: its count in the unit of its own type."""
        return lit(literal_in(e.value, unit_of(ttype(e)))) if is_lit(e) else e

    def rewrite(e: Any) -> Any:  # noqa: C901
        if not isinstance(e, ColumnExpr):
            return e
        if is_lit(e):
            return e
        if e.has_args:
            e = ColumnExpr(e.kind, e.head, [rewrite(a) for a in e.args], e.kwargs, e.is_distinct, e.as_name, e.as_type)
        bare = e.cast(None).alias("") if (e.as_type is not None or e.as_name != "") else e
        out = e
        if e.kind == Kind.BINARY and (is_lit(e.left) or is_lit(e.right)) and not (is_lit(e.left) and is_lit(e.right)):
            x, l, left = (e.right, e.left, True) if is_lit(e.left) else (e.left, e.right, False)
            unit = unit_of(ttype(x))
            if e.head in ("+", "-"):
                k = lit(literal_in(l.value, unit))
                out = ColumnExpr(Kind.BINARY, e.head, [k, x] if left else [x, k], None, False, e.as_name, e.as_type)
                if isinstance(l.value, datetime.timedelta):
                    rows = values(out.cast(None).alias(""))
                    return finish(column([None if v is None else wrap(v) for v in rows], "Int64", e, ttype(x), False), e,
                                  ttype(x))
                return out
            op = _FLIP[e.head] if left else e.head
            out = column([compare(op, v, unit, l.value) for v in values(x)], "boolean", e, None)
            return out
        if e.kind == Kind.CALL and e.head.upper() in ("COALESCE", "GREATEST", "LEAST", "CASE"):
            res = [i for i in range(len(e.args)) if e.head.upper() != "CASE" or i % 2 == 1 or i == len(e.args) - 1]
            if any(is_lit(e.args[i]) for i in res):
                tps = [ttype(e.args[i]) for i in res if not is_lit(e.args[i]) and ttype(e.args[i]) is not None]
                tp = tps[0] if tps else ttype([e.args[i] for i in res if is_lit(e.args[i])][0])
                args = [lit(literal_in(a.value, unit_of(tp))) if (i in res and is_lit(a)) else a
                        for i, a in enumerate(e.args)]
                return ColumnExpr(e.kind, e.head, args, e.kwargs, e.is_distinct, e.as_name, e.as_type)
        if e.kind == Kind.CALL and e.head.upper() in _FUNCS:
            fn = e.head.upper()
            a0 = e.args[0]
            u0 = unit_of(ttype(a0))
            v0 = values(plain(a0))
            if fn == "EXTRACT":
                f = e.kwargs["field"].lower()
                out = column([extract(f, v, u0) for v in v0], "Float64" if f == "epoch" else "Int64", e, None)
            elif fn == "DATE_TRUNC":
                out = column([date_trunc(e.kwargs["part"].lower(), v, u0) for v in v0], "Int64", e, ttype(a0), False)
                return finish(out, e, ttype(a0))
            elif fn == "DATEDIFF":
                v1, u1 = values(plain(e.args[1])), unit_of(ttype(e.args[1]))
                out = column([datediff(e.kwargs["part"].lower(), a, u0, b, u1) for a, b in zip(v0, v1)], "Int64", e, None)
            else:
                ns = values(e.args[1] if isinstance(e.args[1], ColumnExpr) else lit(e.args[1]))
                out = column([add_months(v, k, u0) for v, k in zip(v0, ns)], "Int64", e, ttype(a0), False)
                return finish(out, e, ttype(a0))
            return out
        if e.as_type is not None and unit_of(e.as_type) is not None:
            src = ttype(bare)
            if src is not None and unit_of(src) != unit_of(e.as_type):
                return finish(col(bare.name) if bare.kind == Kind.NAMED else bare, e, src)
        return out

    def finish(rep: Any, e: Any, src: Optional[pa.DataType]) -> Any:
        """Apply a temporal cast of ``e`` to the replacement ``rep`` (a value of type ``src``)."""
        if e.as_type is not None and unit_of(e.as_type) is not None and src is not None and \
                unit_of(src) != unit_of(e.as_type):
            rows = [cast(v, unit_of(src), unit_of(e.as_type)) for v in values(plain(rep.alias("")))]
            name = f"__tm{len(added)}"
            df[name] = pd.array([pd.NA if v is None else v for v in rows], dtype="Int64")
            added.append(name)
            types[name] = e.as_type
            rep = col(name)
            return rep.alias(e.as_name) if e.as_name != "" else rep
        if e.as_type is not None and unit_of(e.as_type) is not None and e.kind != Kind.NAMED:
            types[rep.output_name or rep.name] = e.as_type
        return rep

    out = []
    for e in exprs:
        r = rewrite(e)
        out.append(plain(r) if is_lit(r) else r)
    return df, out, added
