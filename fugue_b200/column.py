"""Column expressions of ``ExecutionEngine.select / filter / assign / aggregate``: the engine's own IR.

One immutable node type (:class:`ColumnExpr`) tagged with a :class:`Kind`; everything the engine needs
from an expression is a function of ``(kind, head, args)``:

    NAMED     head = column name                     WILDCARD  ``*``
    LITERAL   head = python value (None = NULL)      UNARY     head in ``- ~ IS_NULL NOT_NULL``, one arg
    BINARY    head in ``+ - * / & | < > <= >= == !=``  CALL      head = function name (``COALESCE`` ...)
    AGG       head in ``SUM COUNT AVG MIN MAX FIRST LAST``, one arg, optional DISTINCT
    WINDOW    head in the AGG functions (one arg, kwargs ``running``), ``ROW_NUMBER RANK DENSE_RANK`` (no
              arg) or ``LAG LEAD`` (one arg, kwargs ``n`` and ``default``): evaluated over the logical
              partitions of ``fa.transform`` (PartitionSpec keys, presort order) by a ``ColumnMap``

plus an optional output alias and an optional cast of the node's result.  ``fugue_b200/expr.py`` compiles
these trees into programs for the device evaluator (``fb_eval_expr``); nothing goes through SQL text.

The builders keep the names and the observable behaviour (alias / type inference, group-key rules,
error types, string forms) of the reference's public expression interface, so that code written
against ``fugue.column`` reads the same here: ``col, lit, null, all_cols, function`` and the operators
(fugue/column/expressions.py:8-856), ``functions.*`` (fugue/column/functions.py:13-370),
``SelectColumns`` (fugue/column/sql.py:38-246).  The reference's own trees reach the engine through
``fugue_b200.fugue_plugin.translate_expr``; tests/test_column_golden.py pins this module to vectors
produced by the reference's code.
"""
import enum
import hashlib
from typing import Any, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import pyarrow as pa

from .schema import Schema, parse_type, type_to_expr


class Kind(enum.IntEnum):
    NAMED = 0
    WILDCARD = 1
    LITERAL = 2
    UNARY = 3
    BINARY = 4
    CALL = 5
    AGG = 6
    WINDOW = 7


BOOL_OPS = frozenset(["&", "|", "<", ">", "<=", ">=", "==", "!="])
ARITH_OPS = frozenset(["+", "-", "*", "/"])
AGG_KEEPS_ARG_TYPE = frozenset(["MIN", "MAX", "FIRST", "LAST"])
WINDOW_AGGS = frozenset(["SUM", "COUNT", "AVG", "MIN", "MAX", "FIRST", "LAST"])
_RANKINGS = frozenset(["ROW_NUMBER", "RANK", "DENSE_RANK"])
_RUNNING_FRAME = "ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW"
_LITERAL_TYPES = (int, bool, float, str)


def to_pa_datatype(obj: Any) -> pa.DataType:
    """python type / type expression / pyarrow type -> pyarrow type (``int`` -> int64, ``float`` ->
    float64, ``str`` -> string, ``bool`` -> bool; strings follow the schema expression syntax, so
    ``"int"`` -> int32)."""
    import datetime

    if isinstance(obj, pa.DataType):
        return obj
    if isinstance(obj, str):
        return parse_type(obj)
    table = {int: pa.int64(), float: pa.float64(), str: pa.string(), bool: pa.bool_(),
             datetime.datetime: pa.timestamp("us"), datetime.date: pa.date32()}
    if obj in table:
        return table[obj]
    raise TypeError(f"can't convert {obj!r} to a data type")


def _show_arg(v: Any) -> str:
    if isinstance(v, bool):
        return "TRUE" if v else "FALSE"
    if isinstance(v, str):
        return f"'{v}'"
    return str(v)


def _show_literal(v: Any) -> str:
    if v is None:
        return "NULL"
    if isinstance(v, bool):
        return "TRUE" if v else "FALSE"
    if isinstance(v, str):
        return "'" + v.replace("\\", "\\\\").replace("'", "\\'") + "'"
    return str(v)


class ColumnExpr:
    """One node of an expression tree (see the module docstring).  Immutable: ``alias`` / ``cast``
    return modified copies."""

    __slots__ = ("kind", "head", "args", "kwargs", "is_distinct", "as_name", "as_type")

    def __init__(self, kind: Kind, head: Any, args: Sequence[Any] = (), kwargs: Optional[Dict[str, Any]] = None,
                 distinct: bool = False, as_name: str = "", as_type: Optional[pa.DataType] = None):
        self.kind = kind
        self.head = head
        self.args: Tuple[Any, ...] = tuple(args)
        self.kwargs: Dict[str, Any] = dict(kwargs or {})
        self.is_distinct = distinct
        self.as_name = as_name
        self.as_type = as_type

    # ---- accessors (one per role of ``head`` / ``args``) ----------------------------------------
    @property
    def name(self) -> str:
        """Column name of a NAMED node, ``*`` for the wildcard, empty otherwise."""
        if self.kind == Kind.NAMED:
            return self.head
        return "*" if self.kind == Kind.WILDCARD else ""

    @property
    def value(self) -> Any:
        assert self.kind == Kind.LITERAL
        return self.head

    @property
    def op(self) -> str:
        assert self.kind in (Kind.UNARY, Kind.BINARY)
        return self.head

    @property
    def func(self) -> str:
        assert self.kind in (Kind.UNARY, Kind.BINARY, Kind.CALL, Kind.AGG, Kind.WINDOW)
        return self.head

    @property
    def arg(self) -> "ColumnExpr":
        assert self.kind in (Kind.UNARY, Kind.AGG, Kind.WINDOW) and len(self.args) == 1
        return self.args[0]

    col = arg  # operand of a unary operator

    @property
    def left(self) -> "ColumnExpr":
        assert self.kind == Kind.BINARY
        return self.args[0]

    @property
    def right(self) -> "ColumnExpr":
        assert self.kind == Kind.BINARY
        return self.args[1]

    @property
    def has_args(self) -> bool:
        return self.kind in (Kind.UNARY, Kind.BINARY, Kind.CALL, Kind.AGG, Kind.WINDOW)

    @property
    def output_name(self) -> str:
        if self.kind == Kind.WILDCARD:
            raise NotImplementedError("wildcard column doesn't have an output name")
        return self.as_name if self.as_name != "" else self.name

    # ---- derived copies ---------------------------------------------------------------------------
    def _with(self, as_name: str, as_type: Optional[pa.DataType]) -> "ColumnExpr":
        return ColumnExpr(self.kind, self.head, self.args, self.kwargs, self.is_distinct, as_name, as_type)

    def alias(self, as_name: str) -> "ColumnExpr":
        if self.kind == Kind.WILDCARD:
            raise NotImplementedError("wildcard column can't have an alias")
        return self._with(as_name, self.as_type)

    def cast(self, data_type: Any) -> "ColumnExpr":
        if self.kind == Kind.WILDCARD:
            raise NotImplementedError("wildcard column can't be cast")
        return self._with(self.as_name, None if data_type is None else to_pa_datatype(data_type))

    def infer_alias(self) -> "ColumnExpr":
        """Give the node the name SQL would give it: a cast column keeps its name, a unary operator or
        an aggregation of a named column takes the column's name."""
        if self.kind == Kind.NAMED:
            return self.alias(self.head) if (self.as_name == "" and self.as_type is not None) else self
        if self.kind in (Kind.UNARY, Kind.AGG) and self.as_name == "":
            return self.alias(self.args[0].infer_alias().output_name)
        if self.kind == Kind.WINDOW and self.as_name == "" and self.args and self.args[0].kind != Kind.WILDCARD:
            return self.alias(self.args[0].infer_alias().output_name)
        return self

    def infer_type(self, schema: Schema) -> Optional[pa.DataType]:
        """The result type where it follows from the tree alone (None: the evaluator decides)."""
        if self.as_type is not None:
            return self.as_type
        k = self.kind
        if k == Kind.NAMED:
            return schema[self.head].type if self.head in schema else None
        if k == Kind.LITERAL:
            return None if self.head is None else to_pa_datatype(type(self.head))
        if k == Kind.BINARY:
            return pa.bool_() if self.head in BOOL_OPS else None
        if k == Kind.UNARY and self.head in ("-", "~"):
            tp = self.args[0].infer_type(schema)
            if tp is None:
                return None
            fits = (pa.types.is_signed_integer(tp) or pa.types.is_floating(tp)) if self.head == "-" \
                else pa.types.is_boolean(tp)
            return tp if fits else None
        if k == Kind.AGG and self.head in AGG_KEEPS_ARG_TYPE:
            return self.args[0].infer_type(schema)
        if k == Kind.WINDOW:
            if self.head in _RANKINGS or self.head == "COUNT":
                return pa.int64()
            if self.head == "AVG":
                return pa.float64()
            tp = self.args[0].infer_type(schema)
            if self.head == "SUM" and tp is not None:
                return pa.float64() if pa.types.is_floating(tp) else pa.int64()
            return tp  # SUM of an unknown type: None; MIN MAX FIRST LAST LAG LEAD keep the argument's type
        return None

    # ---- text -------------------------------------------------------------------------------------
    def _body(self) -> str:
        k = self.kind
        if k == Kind.NAMED:
            return self.head
        if k == Kind.WILDCARD:
            return "*"
        if k == Kind.LITERAL:
            return _show_literal(self.head)
        if k == Kind.WINDOW:
            return _window_text(self, _show_arg)
        parts = [_show_arg(x) for x in self.args] + [n + "=" + _show_arg(v) for n, v in self.kwargs.items()]
        return f"{self.head}({'DISTINCT ' if self.is_distinct else ''}{','.join(parts)})"

    def __str__(self) -> str:
        res = self._body()
        if self.as_type is not None:
            res = f"CAST({res} AS {type_to_expr(self.as_type)})"
        return res if self.as_name == "" else res + " AS " + self.as_name

    __repr__ = __str__

    def fingerprint(self) -> str:
        """Stable id of the tree (structure, aliases, casts): equal trees get equal temporaries."""
        return hashlib.sha1(_canon(self).encode()).hexdigest()

    # ---- operators --------------------------------------------------------------------------------
    def is_null(self) -> "ColumnExpr":
        if self.kind == Kind.LITERAL:
            return lit(self.head is None)
        return ColumnExpr(Kind.UNARY, "IS_NULL", [self])

    def not_null(self) -> "ColumnExpr":
        if self.kind == Kind.LITERAL:
            return lit(self.head is not None)
        return ColumnExpr(Kind.UNARY, "NOT_NULL", [self])

    def __neg__(self) -> "ColumnExpr":
        return ColumnExpr(Kind.UNARY, "-", [self])

    def __pos__(self) -> "ColumnExpr":
        return self

    def __invert__(self) -> "ColumnExpr":
        return ColumnExpr(Kind.UNARY, "~", [self])

    def over(self, running: bool = False) -> "ColumnExpr":
        """The aggregation as a window function of a ``ColumnMap``: over the whole logical partition
        (``running=False``, the value repeated on every row) or over the rows up to and including the
        current one in presort order (``running=True``)."""
        if self.kind != Kind.AGG:
            raise ValueError(f"{self} is not an aggregation: only an aggregation has an OVER form")
        if self.is_distinct:
            raise ValueError(f"{self}: DISTINCT aggregations have no window form")
        if self.head not in WINDOW_AGGS:
            raise ValueError(f"{self}: {self.head} has no window form")
        if not isinstance(running, bool):
            raise ValueError(f"running must be a bool, got {running!r}")
        if is_agg(self.args[0]) or has_window(self.args[0]):
            raise ValueError(f"nested aggregation {self}")
        if self.head in ("FIRST", "LAST") and self.args[0].kind == Kind.WILDCARD:
            raise ValueError(f"{self}: {self.head} needs a column")
        return ColumnExpr(Kind.WINDOW, self.head, self.args, {"running": running}, False, self.as_name, self.as_type)

    def __bool__(self) -> bool:
        raise TypeError("a column expression has no truth value; use & | ~ to combine conditions")

    __hash__ = object.__hash__


def _binary_method(op: str, swap: bool) -> Any:
    def method(self: ColumnExpr, other: Any) -> ColumnExpr:
        return binary(op, other, self) if swap else binary(op, self, other)

    return method


for _name, _op in (("add", "+"), ("sub", "-"), ("mul", "*"), ("truediv", "/"), ("and", "&"), ("or", "|")):
    setattr(ColumnExpr, f"__{_name}__", _binary_method(_op, False))
    setattr(ColumnExpr, f"__r{_name}__", _binary_method(_op, True))
for _name, _op in (("lt", "<"), ("gt", ">"), ("le", "<="), ("ge", ">="), ("eq", "=="), ("ne", "!=")):
    setattr(ColumnExpr, f"__{_name}__", _binary_method(_op, False))


def _canon(v: Any) -> str:
    if isinstance(v, ColumnExpr):
        inner = ",".join(_canon(a) for a in v.args) + ";" + ",".join(k + "=" + _canon(x) for k, x in v.kwargs.items())
        return (f"<{int(v.kind)}|{type(v.head).__name__}:{v.head!r}|{inner}|{int(v.is_distinct)}|{v.as_name}|"
                f"{v.as_type}>")
    return f"{type(v).__name__}:{v!r}"


# ---- builders -------------------------------------------------------------------------------------
def lit(obj: Any, alias: str = "") -> ColumnExpr:
    if not (obj is None or isinstance(obj, _LITERAL_TYPES)):
        raise NotImplementedError(f"{obj}, type: {type(obj)}")
    return ColumnExpr(Kind.LITERAL, obj, as_name=alias)


def null() -> ColumnExpr:
    return lit(None)


def all_cols() -> ColumnExpr:
    return ColumnExpr(Kind.WILDCARD, "*")


def col(obj: Any, alias: str = "") -> ColumnExpr:
    if isinstance(obj, ColumnExpr):
        return obj if alias == "" else obj.alias(alias)
    if isinstance(obj, str):
        return all_cols() if obj == "*" else ColumnExpr(Kind.NAMED, obj, as_name=alias)
    raise NotImplementedError(obj)


def _operand(obj: Any) -> ColumnExpr:
    return obj if isinstance(obj, ColumnExpr) else lit(obj)


def binary(op: str, left: Any, right: Any) -> ColumnExpr:
    return ColumnExpr(Kind.BINARY, op, [_operand(left), _operand(right)])


def function(name: str, *args: Any, arg_distinct: bool = False, **kwargs: Any) -> ColumnExpr:
    return ColumnExpr(Kind.CALL, name, args, kwargs, arg_distinct)


def agg(func: str, arg: Any, as_name: str = "", arg_distinct: bool = False) -> ColumnExpr:
    """``FUNC([DISTINCT] arg)``: SUM / COUNT / AVG / MIN / MAX / FIRST / LAST."""
    return ColumnExpr(Kind.AGG, func.upper(), [col(arg)], None, arg_distinct, as_name)


def is_agg(column: Any) -> bool:
    """True when the expression contains an aggregation anywhere."""
    if not isinstance(column, ColumnExpr):
        return False
    if column.kind == Kind.AGG:
        return True
    if column.kind == Kind.WINDOW:  # a window function is evaluated per row: not a GROUP BY aggregation
        return False
    return any(is_agg(x) for x in column.args) or any(is_agg(x) for x in column.kwargs.values())


def has_window(column: Any) -> bool:
    """True when the expression contains a window function anywhere."""
    if not isinstance(column, ColumnExpr):
        return False
    if column.kind == Kind.WINDOW:
        return True
    return any(has_window(x) for x in column.args) or any(has_window(x) for x in column.kwargs.values())


def _window_text(e: ColumnExpr, show: Any) -> str:
    """``FUNC(args) OVER (frame)`` of a WINDOW node; ``show`` renders one argument."""
    parts = [show(x) for x in e.args]
    if e.head in ("LAG", "LEAD"):
        parts += [str(e.kwargs["n"]), _show_literal(e.kwargs["default"])]
    frame = _RUNNING_FRAME if e.kwargs.get("running", False) else ""
    return f"{e.head}({','.join(parts)}) OVER ({frame})"


def _offset_fn(name: str, c: Any, n: Any, default: Any) -> ColumnExpr:
    if isinstance(n, bool) or not isinstance(n, int) or n < 0:
        raise ValueError(f"{name}: n must be a non-negative int, got {n!r}")
    if not (default is None or isinstance(default, _LITERAL_TYPES)):
        raise ValueError(f"{name}: default must be a literal or None, got {default!r}")
    arg = col(c)
    if arg.kind == Kind.WILDCARD or is_agg(arg) or has_window(arg):
        raise ValueError(f"{name} needs a row-wise column expression, got {arg}")
    return ColumnExpr(Kind.WINDOW, name, [arg], {"n": n, "default": default})


def column_mentions(column: Any) -> Iterator[str]:
    """Names of the columns an expression reads."""
    if isinstance(column, ColumnExpr):
        if column.kind == Kind.NAMED:
            yield column.head
        for a in column.args:
            yield from column_mentions(a)
        for a in column.kwargs.values():
            yield from column_mentions(a)


class functions:
    """``f = fugue_b200.column.functions`` plays the role of ``import fugue.column.functions as f``."""

    @staticmethod
    def coalesce(*args: Any) -> ColumnExpr:
        return function("COALESCE", *[_operand(x) for x in args])

    @staticmethod
    def min(c: Any) -> ColumnExpr:  # noqa: A003
        return agg("MIN", c)

    @staticmethod
    def max(c: Any) -> ColumnExpr:  # noqa: A003
        return agg("MAX", c)

    @staticmethod
    def first(c: Any) -> ColumnExpr:
        return agg("FIRST", c)

    @staticmethod
    def last(c: Any) -> ColumnExpr:
        return agg("LAST", c)

    @staticmethod
    def count(c: Any) -> ColumnExpr:
        return agg("COUNT", c)

    @staticmethod
    def count_distinct(c: Any) -> ColumnExpr:
        return agg("COUNT", c, arg_distinct=True)

    @staticmethod
    def avg(c: Any) -> ColumnExpr:
        return agg("AVG", c)

    @staticmethod
    def sum(c: Any) -> ColumnExpr:  # noqa: A003
        return agg("SUM", c)

    mean = avg
    is_agg = staticmethod(is_agg)

    @staticmethod
    def row_number() -> ColumnExpr:
        """1, 2, ... in presort order inside every logical partition of ``fa.transform``."""
        return ColumnExpr(Kind.WINDOW, "ROW_NUMBER")

    @staticmethod
    def rank() -> ColumnExpr:
        """SQL RANK: the row number of the first of the current row's peers (equal on every presort column)."""
        return ColumnExpr(Kind.WINDOW, "RANK")

    @staticmethod
    def dense_rank() -> ColumnExpr:
        """SQL DENSE_RANK: 1 + the number of distinct peer groups before the current row's."""
        return ColumnExpr(Kind.WINDOW, "DENSE_RANK")

    @staticmethod
    def lag(c: Any, n: int = 1, default: Any = None) -> ColumnExpr:
        """``c`` of the row ``n`` rows earlier in the same logical partition, else ``default``."""
        return _offset_fn("LAG", c, n, default)

    @staticmethod
    def lead(c: Any, n: int = 1, default: Any = None) -> ColumnExpr:
        """``c`` of the row ``n`` rows later in the same logical partition, else ``default``."""
        return _offset_fn("LEAD", c, n, default)


# ---- one SELECT list ------------------------------------------------------------------------------
class SelectColumns:
    """The output columns of one SELECT, sorted into the roles the engine cares about.  With an
    aggregation present every other non-literal column is a GROUP BY key (stripped of alias and cast)."""

    def __init__(self, *cols: ColumnExpr, arg_distinct: bool = False):
        self.is_distinct = arg_distinct
        self.all_cols: List[ColumnExpr] = [c.infer_alias() for c in cols]
        by_role: Dict[str, List[ColumnExpr]] = {"literal": [], "simple": [], "func": [], "agg": []}
        for c in self.all_cols:
            by_role[self._role(c)].append(c)
        self.literals, self.simple_cols = by_role["literal"], by_role["simple"]
        self.non_agg_funcs, self.agg_funcs = by_role["func"], by_role["agg"]
        self._wildcards = sum(1 for c in self.simple_cols if c.kind == Kind.WILDCARD)
        if self._wildcards > 1:
            raise ValueError("'*' can be used at most once")
        self.group_keys: List[ColumnExpr] = []
        if self.agg_funcs:
            if self._wildcards:
                raise ValueError(f"'*' can't be used in aggregation: {self}")
            self.group_keys = [c.alias("").cast(None) for c in self.all_cols
                               if self._role(c) in ("simple", "func")]

    @staticmethod
    def _role(c: ColumnExpr) -> str:
        if c.kind == Kind.LITERAL:
            return "literal"
        if c.kind in (Kind.NAMED, Kind.WILDCARD):
            return "simple"
        return "agg" if is_agg(c) else "func"

    def __str__(self) -> str:
        return "[" + ", ".join(str(x) for x in self.all_cols) + "]"

    def fingerprint(self) -> str:
        return hashlib.sha1((str(self.is_distinct) + "|".join(_canon(c) for c in self.all_cols)).encode()).hexdigest()

    def replace_wildcard(self, schema: Schema) -> "SelectColumns":
        out: List[ColumnExpr] = []
        for c in self.all_cols:
            out.extend([col(n) for n in schema.names] if c.kind == Kind.WILDCARD else [c])
        return SelectColumns(*out, arg_distinct=self.is_distinct)

    def assert_all_with_names(self) -> "SelectColumns":
        seen = set()
        for x in self.all_cols:
            if x.kind == Kind.WILDCARD:
                continue
            if x.kind == Kind.NAMED and self._wildcards and x.as_name == "":
                raise ValueError(f"with '*', all other columns must have an alias: {self}")
            if x.output_name == "":
                raise ValueError(f"{x} does not have an alias: {self}")
            if x.output_name in seen:
                raise ValueError(f"{x} can't be reused in select: {self}")
            seen.add(x.output_name)
        return self

    def assert_no_wildcard(self) -> "SelectColumns":
        assert self._wildcards == 0
        return self

    def assert_no_agg(self) -> "SelectColumns":
        assert not self.has_agg
        return self

    @property
    def has_agg(self) -> bool:
        return len(self.agg_funcs) > 0

    @property
    def has_literals(self) -> bool:
        return len(self.literals) > 0

    @property
    def simple(self) -> bool:
        return len(self.simple_cols) == len(self.all_cols)


# ---- SQL text of a tree (error messages, INTEGRATION.md examples, the golden test) ------------------
_SQL_OF_OP = {"&": " AND ", "|": " OR ", "==": "="}


def _quote(name: str) -> str:
    plain = name != "" and (name[0].isalpha() or name[0] == "_") and all(ch.isalnum() or ch == "_" for ch in name)
    return name if plain else "`" + name.replace("`", "``") + "`"


def to_sql(expr: ColumnExpr, enable_cast: bool = True, nested: bool = False) -> str:
    """The expression as SQL text (infix operators, ``CAST(.. AS ..)``, back-quoted odd names)."""
    k = expr.kind
    if k == Kind.LITERAL:
        body = _show_literal(expr.head)
    elif k == Kind.NAMED:
        body = _quote(expr.head)
    elif k == Kind.WILDCARD:
        body = "*"
    elif k == Kind.UNARY:
        inner = to_sql(expr.args[0], enable_cast, True)
        body = {"-": "-" + inner, "~": "NOT " + inner, "IS_NULL": inner + " IS NULL",
                "NOT_NULL": inner + " IS NOT NULL"}[expr.head]
    elif k == Kind.WINDOW:
        body = _window_text(expr, lambda x: to_sql(_operand(x), enable_cast))
    elif k == Kind.BINARY:
        if expr.head not in BOOL_OPS and expr.head not in ARITH_OPS:
            raise NotImplementedError(expr)
        body = to_sql(expr.args[0], enable_cast, True) + _SQL_OF_OP.get(expr.head, expr.head) + \
            to_sql(expr.args[1], enable_cast, True)
        if nested:
            body = "(" + body + ")"
    else:
        parts = [to_sql(_operand(x), enable_cast) for x in expr.args] + \
            [n + "=" + to_sql(_operand(v), enable_cast) for n, v in expr.kwargs.items()]
        body = f"{expr.head}({'DISTINCT ' if expr.is_distinct else ''}{','.join(parts)})"
    if enable_cast and expr.as_type is not None:
        body = f"CAST({body} AS {type_to_expr(expr.as_type)})"
    if expr.as_name != "":
        return body + " AS " + _quote(expr.as_name)
    if expr.as_type is not None and expr.name != "":
        return body + " AS " + _quote(expr.name)
    return body


def select_sql(columns: SelectColumns, table: str, where: Optional[ColumnExpr] = None,
               having: Optional[ColumnExpr] = None, enable_cast: bool = True) -> str:
    """``SELECT .. FROM table [WHERE ..] [GROUP BY ..] [HAVING ..]`` for a SELECT list; literals next to
    aggregations are attached by an outer SELECT (they are not group keys)."""
    columns.assert_all_with_names()
    if where is not None and is_agg(where):
        raise ValueError(f"{where} has aggregation functions")
    tail = "" if where is None else " WHERE " + to_sql(where.alias(""), enable_cast)
    head = "SELECT " + ("DISTINCT " if columns.is_distinct else "")
    if columns.has_agg and columns.has_literals:
        inner = SelectColumns(*[x for x in columns.all_cols if x.kind != Kind.LITERAL])
        names = [to_sql(x, enable_cast) if x.kind == Kind.LITERAL else x.output_name for x in columns.all_cols]
        return f"SELECT {', '.join(names)} FROM ( {select_sql(inner, table, where, having, enable_cast)} )"
    text = head + ", ".join(to_sql(x, enable_cast) for x in columns.all_cols) + " FROM " + table + tail
    if columns.has_agg:
        columns.assert_no_wildcard()
        if columns.group_keys:
            text += " GROUP BY " + ", ".join(to_sql(x, enable_cast) for x in columns.group_keys)
        if having is not None:
            text += " HAVING " + to_sql(having.alias(""), enable_cast)
    return text


def correct_select_schema(input_schema: Schema, select: SelectColumns, output_schema: Schema) -> Optional[Schema]:
    """Fields whose inferred type differs from what an evaluator produced (None: nothing to fix)."""
    cols = select.replace_wildcard(input_schema).assert_all_with_names()
    fields = []
    for c in cols.all_cols:
        tp = c.infer_type(input_schema)
        if tp is not None and tp != output_schema[c.output_name].type:
            fields.append(pa.field(c.output_name, tp))
    return Schema(fields) if fields else None
