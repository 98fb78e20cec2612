"""Oracle: the functions that build strings, of one Python string each.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) - never imported by the product path.

SUBSTR, TRIM / LTRIM / RTRIM, REPLACE, CONCAT and ``||`` restate SQLite 3.45 (func.c) in code points, and
tests/test_string_build_cpu.py pins them to the ``sqlite3`` module on random strings.  UPPER / LOWER are
pyarrow's ``utf8_upper`` / ``utf8_lower`` (simple case mapping, one code point to one).  NULL (None) in
gives None out, except that CONCAT skips NULL parts.

``lower_exprs`` turns the string-building nodes of expression trees into columns of their values, then lets
``oracle.strings.lower`` do the same for LIKE / LENGTH, so that ``oracle/expressions.py`` evaluates whole
``select`` / ``filter`` / ``assign`` calls that use them.
"""
import functools
from typing import Any, List, Optional, Tuple

import pyarrow as pa
import pyarrow.compute as pc

from . import strings as ostr

SUBSTR_NO_LENGTH = 1 << 62


@functools.lru_cache(maxsize=1 << 16)
def upper(s: Optional[str]) -> Optional[str]:
    return None if s is None else pc.utf8_upper(pa.array([s], type=pa.string()))[0].as_py()


@functools.lru_cache(maxsize=1 << 16)
def lower(s: Optional[str]) -> Optional[str]:
    return None if s is None else pc.utf8_lower(pa.array([s], type=pa.string()))[0].as_py()


def substr(s: Optional[str], start: Optional[int], length: Any = "absent") -> Optional[str]:
    """SQLite ``substr(s, start[, length])``: 1-based; start 0 is before the first code point; a negative
    start counts from the end; a negative length takes the code points before start."""
    if s is None or start is None or length is None:
        return None
    p1, p2 = start, (SUBSTR_NO_LENGTH if length == "absent" else length)
    neg = p2 < 0
    if neg:
        p2 = -p2
    if p1 < 0:
        p1 += len(s)
        if p1 < 0:
            p2 = max(p2 + p1, 0)
            p1 = 0
    elif p1 > 0:
        p1 -= 1
    elif p2 > 0:
        p2 -= 1
    if neg:
        p1 -= p2
        if p1 < 0:
            p2 += p1
            p1 = 0
    return s[p1:p1 + p2]


def _trim(s: Optional[str], chars: Optional[str], left: bool, right: bool) -> Optional[str]:
    if s is None or chars is None:
        return None
    a, b = 0, len(s)
    while left and a < b and s[a] in chars:
        a += 1
    while right and b > a and s[b - 1] in chars:
        b -= 1
    return s[a:b]


def trim(s: Optional[str], chars: Optional[str] = " ") -> Optional[str]:
    return _trim(s, chars, True, True)


def ltrim(s: Optional[str], chars: Optional[str] = " ") -> Optional[str]:
    return _trim(s, chars, True, False)


def rtrim(s: Optional[str], chars: Optional[str] = " ") -> Optional[str]:
    return _trim(s, chars, False, True)


def replace(s: Optional[str], old: Optional[str], new: Optional[str]) -> Optional[str]:
    """SQLite ``replace``: non-overlapping matches, left to right; an empty ``old`` changes nothing."""
    if s is None or old is None or new is None:
        return None
    return s if old == "" else s.replace(old, new)


def concat(*parts: Optional[str]) -> str:
    return "".join(p for p in parts if p is not None)


def concat_strict(*parts: Optional[str]) -> Optional[str]:
    return None if any(p is None for p in parts) else "".join(parts)


def evaluate(e: Any, value: Optional[str]) -> Optional[str]:
    """A string-building expression over one string column whose value on the row is ``value``."""
    from fugue_b200.column import ColumnExpr, Kind, is_string_build

    if not isinstance(e, ColumnExpr):
        return e
    if e.kind == Kind.NAMED:
        return value
    if e.kind == Kind.LITERAL:
        return e.value
    assert is_string_build(e), e
    args = [evaluate(a, value) for a in e.args]
    if e.kind == Kind.BINARY:
        return concat_strict(*args)
    fn = e.head.upper()
    if fn in ("SUBSTR", "SUBSTRING"):
        return substr(*args)
    return {"UPPER": upper, "LOWER": lower, "TRIM": trim, "LTRIM": ltrim, "RTRIM": rtrim, "REPLACE": replace,
            "CONCAT": concat}[fn](*args)


def lower_exprs(df: Any, exprs: List[Any]) -> Tuple[Any, List[Any], List[str]]:
    """Rewrite the outermost string-building nodes of column expressions into named columns that hold their
    values, and then the LIKE / LENGTH nodes (``oracle.strings.lower``).  Returns the pandas frame with those
    columns added, the rewritten expressions and the names of the added columns.  A replaced node keeps its
    alias and cast."""
    import pandas as pd

    from fugue_b200.column import ColumnExpr, col, column_mentions, is_string_build

    df = df.copy()
    added: List[str] = []
    names = {}

    def rewrite(e: Any) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if is_string_build(e):
            bare = ColumnExpr(e.kind, e.head, e.args, e.kwargs, e.is_distinct)
            key = bare.fingerprint()
            if key not in names:
                names[key] = f"__sb{len(names)}"
                (src,) = set(column_mentions(bare))
                vals = [evaluate(bare, None if x is None or x is pd.NA else x) for x in df[src]]
                df[names[key]] = pd.array(vals, dtype="string")
                added.append(names[key])
            rep = col(names[key])
            rep = rep.cast(e.as_type) if e.as_type is not None else rep
            return rep.alias(e.as_name) if e.as_name != "" else rep
        if e.has_args:
            return ColumnExpr(e.kind, e.head, [rewrite(a) for a in e.args],
                              {k: rewrite(v) for k, v in e.kwargs.items()}, e.is_distinct, e.as_name, e.as_type)
        return e

    out = [rewrite(e) for e in exprs]
    df, out, more = ostr.lower(df, out)
    return df, out, added + more
