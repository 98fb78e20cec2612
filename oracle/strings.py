"""Oracle: LIKE and LENGTH of one Python string, stated through Python's own regular expressions.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) - never imported by the product path.

``like`` translates the pattern character by character into a ``re.fullmatch`` with ``DOTALL``: ``%`` is
``.*``, ``_`` is ``.`` (one code point), with an escape character the next character is a literal, and every
other character is itself.  The match is case-sensitive and covers the whole string.  There is no default
escape character (DuckDB's rule).  ``length`` is the number of code points, ``len`` of a Python string.
NULL (None) in gives None out.  ``lower`` turns the LIKE / LENGTH nodes of expression trees into columns, so that
``oracle/expressions.py`` evaluates whole ``select`` / ``filter`` / ``assign`` calls that use them.
"""
import re
from typing import Any, List, Optional, Tuple


def like_regex(pattern: str, escape: Optional[str] = None) -> "re.Pattern[str]":
    out = []
    i = 0
    while i < len(pattern):
        ch = pattern[i]
        if escape is not None and ch == escape:
            if i + 1 == len(pattern):
                raise ValueError(f"LIKE pattern {pattern!r} ends in the escape character {escape!r}")
            out.append(re.escape(pattern[i + 1]))
            i += 2
            continue
        out.append(".*" if ch == "%" else "." if ch == "_" else re.escape(ch))
        i += 1
    return re.compile("".join(out), re.DOTALL)


def like(value: Optional[str], pattern: str, escape: Optional[str] = None) -> Optional[bool]:
    if value is None:
        return None
    return like_regex(pattern, escape).fullmatch(value) is not None


def length(value: Optional[str]) -> Optional[int]:
    return None if value is None else len(value)


def lower(df: Any, exprs: List[Any]) -> Tuple[Any, List[Any], List[str]]:
    """Rewrite the ``LIKE`` / ``LENGTH`` nodes of column expressions into named columns that hold their values,
    so that ``oracle.expressions`` evaluates the rest.  Returns the pandas frame with those columns added, the
    rewritten expressions (None stays None) and the names of the added columns (for dropping them again).
    A replaced node keeps its alias and cast."""
    import pandas as pd

    from fugue_b200.column import ColumnExpr, Kind, col

    df = df.copy()
    added: List[str] = []
    names = {}

    def value(x: Any) -> Optional[str]:
        return None if x is None or x is pd.NA else x

    def rewrite(e: Any) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if e.kind == Kind.CALL and e.func.upper() in ("LIKE", "LENGTH"):
            bare = ColumnExpr(e.kind, e.head, e.args, e.kwargs, e.is_distinct)
            key = bare.fingerprint()
            if key not in names:
                names[key] = f"__str{len(names)}"
                s = df[e.args[0].name]
                if e.func.upper() == "LIKE":
                    esc = e.args[2].value if len(e.args) > 2 else None
                    rx = like_regex(e.args[1].value, esc)
                    v = pd.array([None if value(x) is None else rx.fullmatch(x) is not None for x in s], dtype="boolean")
                else:
                    v = pd.array([None if value(x) is None else len(x) for x in s], dtype="Int64")
                df[names[key]] = v
                added.append(names[key])
            rep = col(names[key])
            rep = rep.cast(e.as_type) if e.as_type is not None else rep
            return rep.alias(e.as_name) if e.as_name != "" else rep
        if e.has_args:
            return ColumnExpr(e.kind, e.head, [rewrite(a) for a in e.args],
                              {k: rewrite(v) for k, v in e.kwargs.items()}, e.is_distinct, e.as_name, e.as_type)
        return e

    return df, [rewrite(e) for e in exprs], added
