"""Column expressions of ``ExecutionEngine.select / filter / assign / aggregate``: the engine's own IR.

One immutable node type (:class:`ColumnExpr`) tagged with a :class:`Kind`; everything the engine needs
from an expression is a function of ``(kind, head, args)``:

    NAMED     head = column name                     WILDCARD  ``*``
    LITERAL   head = python value (None = NULL)      UNARY     head in ``- ~ IS_NULL NOT_NULL``, one arg
    BINARY    head in ``+ - * / % & | < > <= >= == != ||``  CALL  head = function name (``COALESCE`` ...)
              ``LIKE``: args (string, pattern literal[, escape literal]); ``LENGTH``: args (string,)
              ``CASE``: args (cond1, value1, ..., condN, valueN, else), the ELSE always stored (NULL if absent);
              ``NULLIF ABS FLOOR CEIL SQRT EXP LN LOG10 POWER GREATEST LEAST``; ``ROUND``: args (x, digits literal)
              ``UPPER LOWER``: args (string,); ``SUBSTR``: args (string, start[, length]); ``TRIM LTRIM RTRIM``:
              args (string[, characters]); ``REPLACE``: args (string, from, to); ``CONCAT``: args (part, ...)
              ``EXTRACT``: args (x,), kwarg ``field``; ``DATE_TRUNC``: args (x,), kwarg ``part``; ``DATEDIFF``: args
              (a, b), kwarg ``part``; ``ADD_MONTHS``: args (x, n)
    AGG       head in ``SUM COUNT AVG MIN MAX FIRST LAST VAR_SAMP VAR_POP STDDEV_SAMP STDDEV_POP SKEWNESS
              SKEWNESS_POP KURTOSIS KURTOSIS_POP``, one arg, optional DISTINCT, or ``PERCENTILE_CONT PERCENTILE_DISC``, one arg and kwarg ``q`` (MEDIAN is
              PERCENTILE_CONT at q = 0.5), or ``CORR COVAR_POP COVAR_SAMP REGR_COUNT REGR_AVGX REGR_AVGY
              REGR_SXX REGR_SYY REGR_SXY REGR_SLOPE REGR_INTERCEPT REGR_R2``, two args (a, b) as in SQL: the
              REGR_* functions take the dependent variable y first, (y, x)
    WINDOW    head in the AGG functions (their args, kwargs ``running``, ``rows`` or ``range``; a percentile keeps
              its ``q`` and covers the whole partition; a variance, a shape statistic or a two-argument aggregate takes ``running``
              only), ``ROW_NUMBER RANK
              DENSE_RANK PERCENT_RANK CUME_DIST`` (no arg), ``NTILE`` (no arg, kwarg ``n``), ``LAG LEAD`` (one arg,
              kwargs ``n`` and ``default``) or ``FIRST_VALUE LAST_VALUE NTH_VALUE`` (one arg, NTH_VALUE's kwarg ``n``,
              and the frame kwargs of an aggregate, none for the whole partition): evaluated over the logical
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
import datetime
import enum
import hashlib
import math
from typing import Any, Dict, Iterable, Iterator, List, NamedTuple, Optional, Sequence, Tuple

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
ARITH_OPS = frozenset(["+", "-", "*", "/", "%"])


class Aggregate(NamedTuple):
    """What the engine knows of one aggregate head.  ``family``: ``basic`` (SUM COUNT AVG MIN MAX), ``pick`` (FIRST
    LAST), ``percentile``, ``variance``, ``shape`` (skewness and kurtosis) or ``bivariate``.  ``result``: ``int64``, ``float64``, ``arg`` (the argument's
    type) or ``sum`` (int64, float64 for a float argument).  ``frames``, what ``over()`` takes: ``any`` frame,
    ``running`` (the whole partition or running=True only) or ``none`` (the whole partition only)."""
    family: str
    result: str
    frames: str


# every aggregate head (STDDEV and VARIANCE name the sample forms, SKEW and KURT the bias-corrected shape statistics);
# all of them have a window form.  The variances, the shape statistics and the SQL:2003 binary set functions are
# float64 but REGR_COUNT; x is args[0] of CORR / COVAR_*, args[1] of the
# REGR_* functions (see bivariate_xy)
AGGREGATES: Dict[str, Aggregate] = {
    "SUM": Aggregate("basic", "sum", "any"), "COUNT": Aggregate("basic", "int64", "any"),
    "AVG": Aggregate("basic", "float64", "any"), "MIN": Aggregate("basic", "arg", "any"),
    "MAX": Aggregate("basic", "arg", "any"), "FIRST": Aggregate("pick", "arg", "any"),
    "LAST": Aggregate("pick", "arg", "any"),
    "PERCENTILE_CONT": Aggregate("percentile", "float64", "none"),
    "PERCENTILE_DISC": Aggregate("percentile", "arg", "none"),
    **{h: Aggregate("variance", "float64", "running") for h in ("VAR_SAMP", "VAR_POP", "STDDEV_SAMP", "STDDEV_POP")},
    **{h: Aggregate("shape", "float64", "running") for h in ("SKEWNESS", "SKEWNESS_POP", "KURTOSIS", "KURTOSIS_POP")},
    "REGR_COUNT": Aggregate("bivariate", "int64", "running"),
    **{h: Aggregate("bivariate", "float64", "running")
       for h in ("CORR", "COVAR_POP", "COVAR_SAMP", "REGR_AVGX", "REGR_AVGY", "REGR_SXX", "REGR_SYY", "REGR_SXY",
                 "REGR_SLOPE", "REGR_INTERCEPT", "REGR_R2")},
}
PERCENTILES = frozenset(h for h, a in AGGREGATES.items() if a.family == "percentile")
VARIANCES = frozenset(h for h, a in AGGREGATES.items() if a.family == "variance")
SHAPES = frozenset(h for h, a in AGGREGATES.items() if a.family == "shape")
BIVARIATES = frozenset(h for h, a in AGGREGATES.items() if a.family == "bivariate")
_AGG_ALIASES = {"STDDEV": "STDDEV_SAMP", "VARIANCE": "VAR_SAMP", "SKEW": "SKEWNESS", "KURT": "KURTOSIS"}
_RANKINGS = frozenset(["ROW_NUMBER", "RANK", "DENSE_RANK"])
# window-only heads: NTILE (kwarg ``n``), PERCENT_RANK and CUME_DIST take a spec and no frame; FIRST_VALUE, LAST_VALUE
# and NTH_VALUE (kwarg ``n``) take the frames an aggregate takes.  Neither set belongs to AGGREGATES or SCALARS.
DISTRIBUTIONS = frozenset(["NTILE", "PERCENT_RANK", "CUME_DIST"])
VALUE_HEADS = frozenset(["FIRST_VALUE", "LAST_VALUE", "NTH_VALUE"])
# window-only exponentially weighted heads (pandas' ewm): a spec and no frame, the decay and options as kwargs
EWM_HEADS = frozenset(["EWM_MEAN", "EWM_VAR", "EWM_STD"])
# window heads that take a partition and an order but no frame
_SPEC_ONLY = _RANKINGS | DISTRIBUTIONS | EWM_HEADS | {"LAG", "LEAD"}
_RUNNING_FRAME = "ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW"
_LITERAL_TYPES = (int, bool, float, str, datetime.date, datetime.datetime, datetime.timedelta)
TEMPORAL_LITERALS = (datetime.date, datetime.datetime, datetime.timedelta)
# EXTRACT fields and DATE_TRUNC / DATEDIFF parts, in the order of the device's codes (``epoch`` has no code: it is
# a division of the stored value)
TIME_FIELDS = ("year", "month", "day", "hour", "minute", "second", "quarter", "dow", "isodow", "doy", "week",
               "isoyear")
TIME_PARTS = ("year", "quarter", "month", "week", "day", "hour", "minute", "second")
ROUND_MAX_DIGITS = 18


class Scalar(NamedTuple):
    """What the engine knows of one scalar function head.  ``family``: ``conditional``, ``numeric``, ``string``,
    ``regex`` or ``temporal``.  ``arity``: the least and the most arguments (None: no limit).  ``literals``: the
    Python types of the arguments after the first; each must be a literal of its type or NULL.  ``result``: ``bool``,
    ``int64``, ``float64``, ``string`` (it builds a string from one string expression), ``extract`` (float64 for the
    ``epoch`` field, else int64), ``operand`` (the type of args[0]), ``case`` (string when every result is a string
    literal or NULL) or None (the evaluator decides)."""
    family: str
    arity: Tuple[int, Optional[int]]
    literals: Tuple[type, ...] = ()
    result: Optional[str] = None


# every scalar function head the device evaluates, in its canonical spelling.  NULLIF runs as a CASE and MOD as
# ``%``; EXTRACT, DATE_TRUNC and DATEDIFF take their field or part as a keyword argument
SCALARS: Dict[str, Scalar] = {
    "CASE": Scalar("conditional", (3, None), result="case"), "NULLIF": Scalar("conditional", (2, 2), result="case"),
    "COALESCE": Scalar("conditional", (1, None)), "GREATEST": Scalar("conditional", (2, None)),
    "LEAST": Scalar("conditional", (2, None)),
    **{h: Scalar("numeric", (1, 1)) for h in ("ABS", "FLOOR", "CEIL")},
    "ROUND": Scalar("numeric", (1, 2), (int,)), "MOD": Scalar("numeric", (2, 2)),
    **{h: Scalar("numeric", (1, 1), result="float64") for h in ("SQRT", "EXP", "LN", "LOG10")},
    "POWER": Scalar("numeric", (2, 2), result="float64"),
    "LIKE": Scalar("string", (2, 3), result="bool"), "LENGTH": Scalar("string", (1, 1), result="int64"),
    **{h: Scalar("string", (1, 1), result="string") for h in ("UPPER", "LOWER")},
    "SUBSTR": Scalar("string", (2, 3), (int, int), "string"),
    **{h: Scalar("string", (1, 2), (str,), "string") for h in ("TRIM", "LTRIM", "RTRIM")},
    "REPLACE": Scalar("string", (3, 3), (str, str), "string"), "CONCAT": Scalar("string", (1, None), result="string"),
    **{h: Scalar("regex", (2, 2), result="bool") for h in ("REGEXP_MATCHES", "REGEXP_FULL_MATCH")},
    "REGEXP_EXTRACT": Scalar("regex", (2, 3), (str, int), "string"),
    "REGEXP_REPLACE": Scalar("regex", (3, 4), (str, str, str), "string"),
    "EXTRACT": Scalar("temporal", (1, 1), result="extract"), "DATE_TRUNC": Scalar("temporal", (1, 1), result="operand"),
    "DATEDIFF": Scalar("temporal", (2, 2), result="int64"), "ADD_MONTHS": Scalar("temporal", (2, 2), result="operand"),
}
# other spellings: (canonical head, the arity they allow; None: the head's)
SCALAR_ALIASES: Dict[str, Tuple[str, Optional[Tuple[int, Optional[int]]]]] = {
    "IFNULL": ("COALESCE", (2, 2)), "IF": ("CASE", (3, 3)), "IIF": ("CASE", (3, 3)), "POW": ("POWER", None),
    "CEILING": ("CEIL", None), "SUBSTRING": ("SUBSTR", None), "REGEXP_LIKE": ("REGEXP_MATCHES", None)}
# regular-expression tests of one string expression: bool
REGEX_PREDICATES = frozenset(h for h, s in SCALARS.items() if s.family == "regex" and s.result == "bool")


def result_type(head: str, arg_type: Optional[pa.DataType]) -> Optional[pa.DataType]:
    """The type of aggregate ``head`` of an argument of type ``arg_type`` (None: unknown, and so is a result that
    depends on it)."""
    rule = AGGREGATES[head].result
    if rule in ("int64", "float64"):
        return pa.type_for_alias(rule)
    if rule == "arg" or arg_type is None:
        return arg_type
    return pa.float64() if pa.types.is_floating(arg_type) else pa.int64()


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
             datetime.datetime: pa.timestamp("us"), datetime.date: pa.date32(), datetime.timedelta: pa.duration("us")}
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
    if isinstance(v, datetime.datetime):
        return f"TIMESTAMP '{v.isoformat(sep=' ')}'"
    if isinstance(v, datetime.date):
        return f"DATE '{v.isoformat()}'"
    if isinstance(v, datetime.timedelta):
        return _interval_text(v)
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
        if self.kind in (Kind.AGG, Kind.WINDOW) and self.head in BIVARIATES:
            return self  # two arguments: no implicit name
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
            if self.head in ("+", "-"):  # a date or timestamp moved by a day-time interval keeps its type
                for x, d in ((self.args[0], self.args[1]), (self.args[1], self.args[0])):
                    if d.kind == Kind.LITERAL and d.as_type is None and isinstance(d.head, datetime.timedelta) and \
                            (self.head == "+" or d is self.args[1]):
                        tp = x.infer_type(schema)
                        return tp if tp is not None and pa.types.is_temporal(tp) else None
            return pa.bool_() if self.head in BOOL_OPS else (pa.string() if self.head == "||" else None)
        if k == Kind.UNARY and self.head in ("-", "~"):
            tp = self.args[0].infer_type(schema)
            if tp is None:
                return None
            fits = (pa.types.is_signed_integer(tp) or pa.types.is_floating(tp)) if self.head == "-" \
                else pa.types.is_boolean(tp)
            return tp if fits else None
        if k in (Kind.AGG, Kind.WINDOW) and self.head in AGGREGATES:
            a = AGGREGATES[self.head]
            if k == Kind.AGG and a.family == "basic" and a.result != "arg":
                return None  # SUM / COUNT / AVG: select() keeps the type the group-by gives them
            return result_type(self.head, self.args[0].infer_type(schema))
        if k == Kind.CALL and scalar_head(self.head) is not None:
            rule = scalar_head(self.head)[1].result
            if rule == "extract":
                return pa.float64() if str(self.kwargs.get("field", "")).lower() == "epoch" else pa.int64()
            if rule == "operand":
                return _operand(self.args[0]).infer_type(schema) if self.args else None
            if rule == "case":
                return pa.string() if case_string_results(self) is not None else None
            return None if rule is None else pa.type_for_alias(rule)
        if k == Kind.WINDOW:
            if self.head in ("PERCENT_RANK", "CUME_DIST") or self.head in EWM_HEADS:
                return pa.float64()
            # LAG LEAD FIRST_VALUE LAST_VALUE NTH_VALUE: the arg's
            return pa.int64() if self.head in _RANKINGS or self.head == "NTILE" else self.args[0].infer_type(schema)
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

    def like(self, pattern: Any, escape: Optional[str] = None) -> "ColumnExpr":
        """SQL ``self LIKE pattern [ESCAPE escape]``: a case-sensitive match of the whole string, ``%`` any
        sequence of characters, ``_`` exactly one character (code point).  No escape character unless one is
        given; with ``escape``, it makes the next character of the pattern a literal."""
        if isinstance(pattern, ColumnExpr) and pattern.kind == Kind.LITERAL and pattern.as_type is None:
            pattern = pattern.value
        if not isinstance(pattern, str):
            raise NotImplementedError(f"LIKE needs a string literal pattern, got {pattern!r}")
        if escape is not None:
            if not isinstance(escape, str) or len(escape) != 1:
                raise ValueError(f"ESCAPE takes exactly one character, got {escape!r}")
            i = 0
            while i < len(pattern):
                if pattern[i] == escape:
                    if i + 1 == len(pattern):
                        raise ValueError(f"LIKE pattern {pattern!r} ends in the escape character {escape!r}")
                    i += 1
                i += 1
        args = [self, lit(pattern)] + ([] if escape is None else [lit(escape)])
        return ColumnExpr(Kind.CALL, "LIKE", args)

    def rlike(self, pattern: Any) -> "ColumnExpr":
        """SQL ``self RLIKE pattern``: ``functions.regexp_matches(self, pattern)``."""
        return functions.regexp_matches(self, pattern)

    def over(self, running: bool = False, rows: Optional[Tuple[Optional[int], Optional[int]]] = None,
             range: Optional[Tuple[Any, Any]] = None,  # noqa: A002 - the SQL word
             partition_by: Optional[Sequence[Any]] = None, order_by: Optional[Sequence[Any]] = None) -> "ColumnExpr":
        """The aggregation as a window function of a ``ColumnMap``: over the whole logical partition
        (``running=False``, the value repeated on every row), over the rows up to and including the
        current one in presort order (``running=True``), over a moving frame ``rows=(start, end)``:
        ``ROWS BETWEEN`` offsets from the current row in presort order, negative PRECEDING, 0 CURRENT ROW,
        positive FOLLOWING, ``None`` UNBOUNDED, or over a value frame ``range=(start, end)``: ``RANGE
        BETWEEN`` offsets in the units of the presort column (``int``, finite ``float`` or
        ``datetime.timedelta``; 0 is CURRENT ROW, the current row's peers).  ``rows=(None, 0)`` is
        ``running=True``, and ``rows=(None, None)`` and ``range=(None, None)`` are the whole partition: they
        give those nodes.  ``range=(None, 0)`` is not ``running=True``: it includes the current row's peers.

        ``partition_by`` (names or expressions) and ``order_by`` (names, expressions or ``(name_or_expr,
        ascending)`` pairs) make the node explicit: it carries its own partition and order, SQL's ``OVER
        (PARTITION BY .. ORDER BY ..)``, and runs in ``select / assign / filter`` and SQL, not in a ``ColumnMap``.
        Either one given, even as ``[]``, makes it explicit; ``partition_by=[]`` alone is ``OVER ()``, the whole
        table.  NULLs sort last in both directions.  The frame keeps the meaning above (the default is the whole
        partition, not SQL's running default of a statement with ORDER BY).  ROW_NUMBER, RANK, DENSE_RANK, NTILE,
        PERCENT_RANK, CUME_DIST, LAG and LEAD take a spec and no frame; a percentile takes ``partition_by`` only;
        FIRST_VALUE, LAST_VALUE and NTH_VALUE take every frame and spec an aggregate takes, once."""
        explicit = partition_by is not None or order_by is not None
        spec = _window_spec(self, partition_by, order_by) if explicit else {}
        if self.kind == Kind.WINDOW and self.head in _SPEC_ONLY and explicit and not is_explicit(self):
            if running or rows is not None or range is not None:
                raise ValueError(f"{self}: {self.head} takes no frame")
            if self.head in EWM_HEADS and self.kwargs["times"]:
                order = spec["order_by"]
                if len(order) != 1:
                    raise ValueError(f"{self}: time decay needs exactly one ORDER BY expression")
                if not order[0][1]:
                    raise ValueError(f"{self}: time decay needs ascending times; ORDER BY is DESC")
            return ColumnExpr(Kind.WINDOW, self.head, self.args, {**self.kwargs, **spec}, False, self.as_name,
                              self.as_type)
        if self.kind == Kind.WINDOW and self.head in VALUE_HEADS:
            if is_explicit(self) or any(k in self.kwargs for k in ("running", "rows", "range")):
                raise ValueError(f"{self} already has its window")
            if not isinstance(running, bool):
                raise ValueError(f"running must be a bool, got {running!r}")
            running, rows, range = _normalise_frame(running, rows, range)
            if explicit and range is not None and any(b not in (None, 0) for b in range) and \
                    len(spec["order_by"]) != 1:
                raise ValueError(f"{self}: a RANGE frame with an offset needs exactly one ORDER BY expression")
            return ColumnExpr(Kind.WINDOW, self.head, self.args, {**self.kwargs, **_frame_kwargs(running, rows, range),
                                                                   **spec}, False, self.as_name, self.as_type)
        if self.kind != Kind.AGG:
            raise ValueError(f"{self} is not an aggregation: only an aggregation has an OVER form")
        if self.is_distinct:
            raise ValueError(f"{self}: DISTINCT aggregations have no window form")
        a = AGGREGATES.get(self.head)
        if a is None:
            raise ValueError(f"{self}: {self.head} has no window form")
        if not isinstance(running, bool):
            raise ValueError(f"running must be a bool, got {running!r}")
        if a.frames == "none":
            if running or rows is not None or range is not None:
                raise ValueError(f"{self}: a percentile covers the whole partition; it takes no frame")
            if spec.get("order_by"):
                raise ValueError(f"{self}: a percentile covers the whole partition; it takes no ORDER BY")
            return ColumnExpr(Kind.WINDOW, self.head, self.args, {**self.kwargs, **spec}, False, self.as_name,
                              self.as_type)
        running, rows, range = _normalise_frame(running, rows, range)
        if a.frames == "running" and (rows is not None or range is not None):
            hint = "; write ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW for the running form" \
                if range == (None, 0) else ""
            raise NotImplementedError(f"{self}: {self.head} runs over the whole partition or running=True; "
                                      f"ROWS and RANGE frames are not supported{hint}")
        # a window over GROUP BY results (explicit only) may read aggregations; nothing reads a window
        if any((is_agg(a) and not explicit) or has_window(a) for a in self.args):
            raise ValueError(f"nested aggregation {self}")
        if a.family == "pick" and self.args[0].kind == Kind.WILDCARD:
            raise ValueError(f"{self}: {self.head} needs a column")
        if explicit and range is not None and any(b not in (None, 0) for b in range) and len(spec["order_by"]) != 1:
            raise ValueError(f"{self}: a RANGE frame with an offset needs exactly one ORDER BY expression")
        return ColumnExpr(Kind.WINDOW, self.head, self.args, {**_frame_kwargs(running, rows, range), **spec}, False,
                          self.as_name, self.as_type)

    def __bool__(self) -> bool:
        raise TypeError("a column expression has no truth value; use & | ~ to combine conditions")

    __hash__ = object.__hash__


def _normalise_frame(running: bool, rows: Any, range: Any) -> Tuple[bool, Any, Any]:  # noqa: A002 - the SQL word
    """The checked frame of ``over()``: ``rows=(None, 0)`` is ``running=True``, ``rows=(None, None)`` and ``range=(None,
    None)`` the whole partition."""
    if range is not None:
        if running or rows is not None:
            raise ValueError("over() takes one of running=True, rows and range")
        range = _range_frame(range)
        if range == (None, None):
            range = None
    if rows is not None:
        if running:
            raise ValueError("over() takes running=True or rows, not both")
        if not isinstance(rows, tuple) or len(rows) != 2:
            raise ValueError(f"rows must be a (start, end) tuple, got {rows!r}")
        for b in rows:
            if isinstance(b, bool) or not (b is None or isinstance(b, int)):
                raise ValueError(f"a frame bound must be an int or None, got {b!r}")
        if rows[0] is not None and rows[1] is not None and rows[0] > rows[1]:
            raise ValueError(f"frame start {rows[0]} is after its end {rows[1]}")
        if rows == (None, 0):
            running, rows = True, None
        elif rows == (None, None):
            rows = None
    return running, rows, range


def _frame_kwargs(running: bool, rows: Any, range: Any) -> Dict[str, Any]:  # noqa: A002 - the SQL word
    if range is not None:
        return {"range": range}
    return {"running": running} if rows is None else {"rows": (rows[0], rows[1])}


def _binary_method(op: str, swap: bool) -> Any:
    def method(self: ColumnExpr, other: Any) -> ColumnExpr:
        return binary(op, other, self) if swap else binary(op, self, other)

    return method


for _name, _op in (("add", "+"), ("sub", "-"), ("mul", "*"), ("truediv", "/"), ("mod", "%"), ("and", "&"),
                   ("or", "|")):
    setattr(ColumnExpr, f"__{_name}__", _binary_method(_op, False))
    setattr(ColumnExpr, f"__r{_name}__", _binary_method(_op, True))
for _name, _op in (("lt", "<"), ("gt", ">"), ("le", "<="), ("ge", ">="), ("eq", "=="), ("ne", "!=")):
    setattr(ColumnExpr, f"__{_name}__", _binary_method(_op, False))


def _canon(v: Any) -> str:
    if isinstance(v, ColumnExpr):
        inner = ",".join(_canon(a) for a in v.args) + ";" + ",".join(k + "=" + _canon(x) for k, x in v.kwargs.items())
        return (f"<{int(v.kind)}|{type(v.head).__name__}:{v.head!r}|{inner}|{int(v.is_distinct)}|{v.as_name}|"
                f"{v.as_type}>")
    if isinstance(v, tuple) and any(isinstance(x, (ColumnExpr, tuple)) for x in v):  # a window spec
        return "(" + ",".join(_canon(x) for x in v) + ")"
    return f"{type(v).__name__}:{v!r}"


# ---- builders -------------------------------------------------------------------------------------
def lit(obj: Any, alias: str = "") -> ColumnExpr:
    """A literal: None (NULL), bool, int, float, str, ``datetime.date`` (date32), ``datetime.datetime`` (timestamp[us];
    a naive one is UTC wall clock, an aware one is converted to UTC) or ``datetime.timedelta`` (duration[us])."""
    if not (obj is None or isinstance(obj, _LITERAL_TYPES)):
        raise NotImplementedError(f"{obj}, type: {type(obj)}")
    if isinstance(obj, datetime.datetime) and obj.tzinfo is not None:
        obj = obj.astimezone(datetime.timezone.utc).replace(tzinfo=None)
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
    """``FUNC([DISTINCT] arg)``: SUM / COUNT / AVG / MIN / MAX / FIRST / LAST / VAR_SAMP / VAR_POP / STDDEV_SAMP /
    STDDEV_POP / SKEWNESS / SKEWNESS_POP / KURTOSIS / KURTOSIS_POP (STDDEV and VARIANCE give the sample forms, SKEW
    and KURT the bias-corrected ones)."""
    func = func.upper()
    return ColumnExpr(Kind.AGG, _AGG_ALIASES.get(func, func), [col(arg)], None, arg_distinct, as_name)


def _bivariate(func: str, a: Any, b: Any) -> ColumnExpr:
    """``FUNC(a, b)`` of ``BIVARIATES``: two row-wise column expressions (or column names)."""
    args = [col(a), col(b)]
    for x in args:
        if x.kind == Kind.WILDCARD or is_agg(x) or has_window(x):
            raise ValueError(f"{func} needs two row-wise column expressions, got {x}")
    return ColumnExpr(Kind.AGG, func, args)


def bivariate_xy(e: ColumnExpr) -> Tuple[ColumnExpr, ColumnExpr]:
    """(x, y) of a ``BIVARIATES`` node: (a, b) of ``CORR / COVAR_*(a, b)``, (x, y) of ``REGR_*(y, x)``."""
    return (e.args[1], e.args[0]) if e.head.startswith("REGR_") else (e.args[0], e.args[1])


def _percentile(func: str, c: Any, q: Any) -> ColumnExpr:
    """``PERCENTILE_CONT / PERCENTILE_DISC(q) WITHIN GROUP (ORDER BY c)``; ``q`` an int or float in [0, 1]."""
    if isinstance(q, bool) or not isinstance(q, (int, float)) or not 0 <= q <= 1:  # NaN fails the range test
        raise ValueError(f"{func}: q must be an int or float in [0, 1], got {q!r}")
    arg = col(c)
    if arg.kind == Kind.WILDCARD or is_agg(arg) or has_window(arg):
        raise ValueError(f"{func} needs a row-wise column expression, got {arg}")
    return ColumnExpr(Kind.AGG, func, [arg], {"q": float(q)})


def _within_group(e: ColumnExpr, show: Any) -> str:
    """``PERCENTILE_CONT(q) WITHIN GROUP (ORDER BY arg)``: the SQL form of a percentile."""
    return f"{e.head}({e.kwargs['q']!r}) WITHIN GROUP (ORDER BY {show(e.args[0])})"


def _children(e: ColumnExpr) -> Iterator[ColumnExpr]:
    """The sub-expressions of a node: its arguments, its keyword arguments and the expressions of a window spec."""
    def walk(v: Any) -> Iterator[ColumnExpr]:
        if isinstance(v, ColumnExpr):
            yield v
        elif isinstance(v, tuple):
            for x in v:
                yield from walk(x)

    for v in list(e.args) + list(e.kwargs.values()):
        yield from walk(v)


def is_agg(column: Any) -> bool:
    """True when the expression contains an aggregation anywhere."""
    if not isinstance(column, ColumnExpr):
        return False
    if column.kind == Kind.AGG:
        return True
    if column.kind == Kind.WINDOW:  # a window function is evaluated per row: not a GROUP BY aggregation
        return False
    return any(is_agg(x) for x in _children(column))


def has_window(column: Any) -> bool:
    """True when the expression contains a window function anywhere."""
    if not isinstance(column, ColumnExpr):
        return False
    if column.kind == Kind.WINDOW:
        return True
    return any(has_window(x) for x in _children(column))


def is_explicit(column: Any) -> bool:
    """True for a window node with its own PARTITION BY / ORDER BY (``over(partition_by=.., order_by=..)``)."""
    return isinstance(column, ColumnExpr) and column.kind == Kind.WINDOW and "partition_by" in column.kwargs


def has_bare_window(column: Any) -> bool:
    """True when the expression contains a window node without a spec: one that only a ``ColumnMap`` evaluates."""
    if not isinstance(column, ColumnExpr):
        return False
    if column.kind == Kind.WINDOW and not is_explicit(column):
        return True
    return any(has_bare_window(x) for x in _children(column))


def has_explicit_window(column: Any) -> bool:
    """True when the expression contains a window node with its own PARTITION BY / ORDER BY."""
    if not isinstance(column, ColumnExpr):
        return False
    return is_explicit(column) or any(has_explicit_window(x) for x in _children(column))


def window_reads_agg(column: Any) -> bool:
    """True when a window function of the expression reads an aggregation: a window over GROUP BY results."""
    if not isinstance(column, ColumnExpr):
        return False
    if column.kind == Kind.WINDOW:
        return any(is_agg(x) for x in _children(column))
    return any(window_reads_agg(x) for x in _children(column))


def _window_spec(e: ColumnExpr, partition_by: Any, order_by: Any) -> Dict[str, Any]:
    """The ``partition_by`` / ``order_by`` kwargs of an explicit window node: a tuple of expressions and a tuple of
    (expression, ascending) pairs, aliases dropped."""
    def item(x: Any) -> ColumnExpr:
        c = col(x) if isinstance(x, (str, ColumnExpr)) else None
        if c is None or c.kind == Kind.WILDCARD or c.kind == Kind.LITERAL:
            raise ValueError(f"{e}: a window partitions and orders by column expressions, got {x!r}")
        if has_window(c):
            raise ValueError(f"{e}: a window function inside another window's PARTITION BY / ORDER BY: {c}")
        return c.alias("")

    for what, v in (("partition_by", partition_by), ("order_by", order_by)):
        if v is not None and (isinstance(v, (str, ColumnExpr)) or not isinstance(v, (list, tuple))):
            raise ValueError(f"{what} must be a list, got {v!r}")
    order = []
    for x in order_by or []:
        if isinstance(x, tuple):
            if len(x) != 2 or not isinstance(x[1], bool):
                raise ValueError(f"an ORDER BY item is a name, an expression or a (name_or_expr, ascending) pair, "
                                 f"got {x!r}")
            order.append((item(x[0]), x[1]))
        else:
            order.append((item(x), True))
    return {"partition_by": tuple(item(x) for x in partition_by or []), "order_by": tuple(order)}


def _window_text(e: ColumnExpr, show: Any) -> str:
    """``FUNC(args) OVER (spec frame)`` of a WINDOW node; ``show`` renders one argument.  A bare node shows its
    frame; an explicit one shows its frame only where it is not SQL's default for its spec (RANGE BETWEEN
    UNBOUNDED PRECEDING AND CURRENT ROW with ORDER BY, the whole partition without), so that its text parses
    back to the same node."""
    spec = []
    if is_explicit(e):
        if e.kwargs["partition_by"]:
            spec.append("PARTITION BY " + ", ".join(show(x) for x in e.kwargs["partition_by"]))
        if e.kwargs["order_by"]:
            spec.append("ORDER BY " + ", ".join(show(x) + ("" if asc else " DESC") for x, asc in e.kwargs["order_by"]))
    if e.head in PERCENTILES:
        return _within_group(e, show) + f" OVER ({' '.join(spec)})"
    parts = [show(x) for x in e.args]
    if e.head in ("LAG", "LEAD"):
        parts += [str(e.kwargs["n"]), _show_literal(e.kwargs["default"])]
    elif e.head in ("NTILE", "NTH_VALUE"):
        parts.append(str(e.kwargs["n"]))
    elif e.head in EWM_HEADS:
        parts += _ewm_text(e.kwargs)
    frame = _RUNNING_FRAME if e.kwargs.get("running", False) else ""
    for unit in ("rows", "range"):
        if unit in e.kwargs:
            frame = f"{unit.upper()} BETWEEN {_frame_bound(e.kwargs[unit][0], 'PRECEDING')} AND " \
                    f"{_frame_bound(e.kwargs[unit][1], 'FOLLOWING')}"
    if is_explicit(e) and e.head not in _SPEC_ONLY:
        default = "RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW" if e.kwargs["order_by"] else ""
        whole = "ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING"
        frame = "" if frame == default else (frame or whole)
    return f"{e.head}({','.join(parts)}) OVER ({' '.join(spec + ([frame] if frame else []))})"


def _ewm_text(kw: Dict[str, Any]) -> List[str]:
    """The arguments after x of an EWM node: SQL's ``alpha [, adjust]`` or ``INTERVAL halflife [, adjust]``, and
    ``name=value`` for what SQL does not spell (com, span, a numeric halflife, ignore_na, min_periods, bias)."""
    key = next(k for k in EWM_DECAYS if k in kw)
    sql = key == "alpha" or (kw["times"] and isinstance(kw[key], datetime.timedelta))
    if sql:
        parts = [_interval_text(kw[key]) if kw["times"] else repr(kw[key])]
    else:
        parts = [f"{key}={kw[key]!r}"] + (["times=TRUE"] if kw["times"] else [])
    if not kw["adjust"]:
        parts.append("FALSE" if sql else "adjust=FALSE")
    if kw["ignore_na"]:
        parts.append("ignore_na=TRUE")
    if kw["min_periods"]:
        parts.append(f"min_periods={kw['min_periods']}")
    if kw.get("bias"):
        parts.append("bias=TRUE")
    return parts


def _frame_bound(b: Any, unbounded: str) -> str:
    if b is None:
        return "UNBOUNDED " + unbounded
    if b == 0:
        return "CURRENT ROW"
    neg = b < (datetime.timedelta(0) if isinstance(b, datetime.timedelta) else 0)
    mag = -b if neg else b
    text = _interval_text(mag) if isinstance(mag, datetime.timedelta) else str(mag)
    return f"{text} PRECEDING" if neg else f"{text} FOLLOWING"


def _interval_text(d: datetime.timedelta) -> str:
    """A timedelta as an SQL day-time INTERVAL literal: ``INTERVAL '7' DAY`` for whole days, else
    ``INTERVAL '1 02:03:04[.000005]' DAY TO SECOND``; a negative one carries one leading ``-`` for the whole value."""
    sign = "-" if d < datetime.timedelta(0) else ""
    d = abs(d)
    if d.seconds == 0 and d.microseconds == 0:
        return f"INTERVAL '{sign}{d.days}' DAY"
    hms = f"{d.seconds // 3600:02d}:{d.seconds // 60 % 60:02d}:{d.seconds % 60:02d}"
    frac = f".{d.microseconds:06d}" if d.microseconds else ""
    return f"INTERVAL '{sign}{d.days} {hms}{frac}' DAY TO SECOND"


def _range_frame(frame: Any) -> Tuple[Any, Any]:
    """Check a ``range=(start, end)`` frame and read a zero bound (``0.0``, ``timedelta(0)``) as the int 0."""
    if not isinstance(frame, tuple) or len(frame) != 2:
        raise ValueError(f"range must be a (start, end) tuple, got {frame!r}")
    out = []
    for b in frame:
        if b is None:
            out.append(None)
            continue
        if isinstance(b, bool) or not isinstance(b, (int, float, datetime.timedelta)):
            raise ValueError(f"a RANGE bound must be an int, a float, a timedelta or None, got {b!r}")
        if isinstance(b, float) and not math.isfinite(b):
            raise ValueError(f"a RANGE bound must be finite, got {b!r}")
        out.append(0 if b == (datetime.timedelta(0) if isinstance(b, datetime.timedelta) else 0) else b)
    start, end = out
    if start is not None and end is not None:
        if isinstance(start, datetime.timedelta) != isinstance(end, datetime.timedelta) and start != 0 and end != 0:
            raise ValueError(f"RANGE bounds mix a timedelta and a number: {frame!r}")
        us = datetime.timedelta(microseconds=1)  # a timedelta as exact integer microseconds
        if (start // us if isinstance(start, datetime.timedelta) else start) > \
                (end // us if isinstance(end, datetime.timedelta) else end):
            raise ValueError(f"frame start {start} is after its end {end}")
    return start, end


def _offset_fn(name: str, c: Any, n: Any, default: Any, aggregated: bool = False) -> ColumnExpr:
    """LAG / LEAD of ``c`` by ``n >= 0`` rows, ``default`` (a literal) where that row is outside the partition.  The
    default is converted to the argument's type as a literal in a CAST would be, when the plan is built, and one the
    type cannot hold exactly (2.5 for an integer, 1000 for int8, -1 for uint64, noon for a date, a string for a number)
    raises ValueError (``colmap.offset_default``, DESIGN §7p); any ``n`` at or past a partition's length gives it."""
    if isinstance(n, bool) or not isinstance(n, int) or n < 0:
        raise ValueError(f"{name}: n must be a non-negative int, got {n!r}")
    if not (default is None or isinstance(default, _LITERAL_TYPES)):
        raise ValueError(f"{name}: default must be a literal or None, got {default!r}")
    arg = col(c)
    if arg.kind == Kind.WILDCARD or (is_agg(arg) and not aggregated) or has_window(arg):
        raise ValueError(f"{name} needs a row-wise column expression, got {arg}")
    return ColumnExpr(Kind.WINDOW, name, [arg], {"n": n, "default": default})


EWM_DECAYS = ("alpha", "com", "span", "halflife")


def _ewm_fn(name: str, c: Any, decay: Dict[str, Any], adjust: Any, ignore_na: Any, min_periods: Any, times: Any,
            bias: Any = None) -> ColumnExpr:
    """An EWM node: ``decay`` the given ones of com / span / halflife / alpha (exactly one), checked as pandas checks
    them; ``times`` a time decay over the node's single order column (``halflife`` only: a ``timedelta`` for a temporal
    column, a positive number for a numeric one)."""
    given = {k: v for k, v in decay.items() if v is not None}
    if len(given) != 1:
        raise ValueError(f"{name}: give exactly one of com, span, halflife and alpha, got {sorted(given) or 'none'}")
    for what, v in (("adjust", adjust), ("ignore_na", ignore_na), ("times", times)) + \
            ((("bias", bias),) if bias is not None else ()):
        if not isinstance(v, bool):
            raise ValueError(f"{name}: {what} must be a bool, got {v!r}")
    if isinstance(min_periods, bool) or not isinstance(min_periods, int) or min_periods < 0:
        raise ValueError(f"{name}: min_periods must be an int >= 0, got {min_periods!r}")
    (key, v), = given.items()
    if times:
        if key != "halflife":
            raise ValueError(f"{name}: time decay takes halflife, not {key}")
        if ignore_na:
            raise NotImplementedError(f"{name}: time decay with ignore_na=True is not supported")
        if name != "EWM_MEAN":
            raise NotImplementedError(f"{name}: time decay is supported for EWM_MEAN only")
    if isinstance(v, datetime.timedelta):
        if not (times and key == "halflife"):
            raise ValueError(f"{name}: a timedelta {key} needs times=True")
        if v <= datetime.timedelta(0):
            raise ValueError(f"{name}: halflife must be > 0, got {v}")
    else:
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
            raise ValueError(f"{name}: {key} must be a finite number, got {v!r}")
        v = float(v) if key != "halflife" or not times or isinstance(v, float) else v
        low = {"alpha": "0 < alpha <= 1", "com": "com >= 0", "span": "span >= 1", "halflife": "halflife > 0"}[key]
        ok = {"alpha": 0 < v <= 1, "com": v >= 0, "span": v >= 1, "halflife": v > 0}[key]
        if not ok:
            raise ValueError(f"{name}: {key} must satisfy {low}, got {v!r}")
    arg = col(c)
    if arg.kind == Kind.WILDCARD or is_agg(arg) or has_window(arg):
        raise ValueError(f"{name} needs a row-wise column expression, got {arg}")
    kw: Dict[str, Any] = {key: v, "adjust": adjust, "ignore_na": ignore_na, "min_periods": min_periods, "times": times}
    if bias is not None:
        kw["bias"] = bias
    return ColumnExpr(Kind.WINDOW, name, [arg], kw)


def ewm_alpha(kw: Dict[str, Any]) -> float:
    """pandas' alpha of an EWM node's decay, in float64 as pandas computes it: through the center of mass, 1 / (1 +
    com).  A time decay runs with pandas' default com = 1 (alpha 0.5): its weights decay by 0.5^(dt / halflife)."""
    if kw["times"]:
        return 0.5
    if "com" in kw:
        com = kw["com"]
    elif "span" in kw:
        com = (kw["span"] - 1) / 2
    elif "halflife" in kw:
        com = 1 / (1 - math.exp(math.log(0.5) / kw["halflife"])) - 1
    else:
        com = (1 - kw["alpha"]) / kw["alpha"]
    return float(1 / (1 + com))


def _nth(name: str, n: Any) -> int:
    if isinstance(n, bool) or not isinstance(n, int) or n < 1:
        raise ValueError(f"{name}: n must be an int >= 1, got {n!r}")
    return n


def _value_fn(name: str, c: Any, kwargs: Dict[str, Any], aggregated: bool = False) -> ColumnExpr:
    """FIRST_VALUE / LAST_VALUE / NTH_VALUE of the row-wise expression ``c`` (over GROUP BY results, ``aggregated``,
    it may read aggregations)."""
    arg = col(c)
    if arg.kind == Kind.WILDCARD or (is_agg(arg) and not aggregated) or has_window(arg):
        raise ValueError(f"{name} needs a row-wise column expression, got {arg}")
    return ColumnExpr(Kind.WINDOW, name, [arg], kwargs)


def scalar_head(name: str) -> Optional[Tuple[str, Scalar]]:
    """The canonical head of scalar function ``name`` (any letter case, any spelling) and its catalogue entry, with
    the narrower arity of an alias; None for a name that is not in ``SCALARS``."""
    up = name.upper()
    if up in SCALAR_ALIASES:
        head, arity = SCALAR_ALIASES[up]
        return head, SCALARS[head] if arity is None else SCALARS[head]._replace(arity=arity)
    return (up, SCALARS[up]) if up in SCALARS else None


def check_arity(name: str, n: int) -> str:
    """The canonical head of ``SCALARS`` function ``name``; ValueError unless it takes ``n`` arguments."""
    head, s = scalar_head(name)
    lo, hi = s.arity
    if n < lo or (hi is not None and n > hi):
        want = str(lo) if lo == hi else f"at least {lo}" if hi is None else f"{lo} to {hi}"
        raise ValueError(f"{name.upper()} takes {want} argument(s), got {n}")
    return head


def check_call(name: str, args: Sequence[Any]) -> Tuple[str, List[ColumnExpr]]:
    """The canonical head and the argument nodes of a call of ``SCALARS`` function ``name``, checked against its
    entry: a wrong number of arguments or a literal of the wrong type raises ValueError, an argument that must be a
    literal and is not raises NotImplementedError."""
    head = check_arity(name, len(args))
    nodes = [_operand(a) for a in args]
    for i, (e, tp) in enumerate(zip(nodes[1:], SCALARS[head].literals)):
        if e.kind != Kind.LITERAL or e.as_type is not None:
            raise NotImplementedError(f"{head}: argument {i + 2} must be a {tp.__name__} literal, got {e}")
        if e.value is not None and (isinstance(e.value, bool) or not isinstance(e.value, tp)):
            raise ValueError(f"{head}: argument {i + 2} must be a {tp.__name__} literal or NULL, got {e.value!r}")
    return head, nodes


def _call(name: str, *args: Any) -> ColumnExpr:
    head, nodes = check_call(name, args)
    return ColumnExpr(Kind.CALL, head, nodes)


def round_digits(d: Any) -> int:
    """The digits of ROUND: an int literal in [-ROUND_MAX_DIGITS, ROUND_MAX_DIGITS], else ValueError."""
    v = d.value if isinstance(d, ColumnExpr) and d.kind == Kind.LITERAL and d.as_type is None else d
    if isinstance(v, bool) or not isinstance(v, int) or not -ROUND_MAX_DIGITS <= v <= ROUND_MAX_DIGITS:
        raise ValueError(f"ROUND takes an integer literal in [-{ROUND_MAX_DIGITS}, {ROUND_MAX_DIGITS}] as its "
                         f"digits, got {d!r}")
    return v


def result_args(e: ColumnExpr) -> List[Any]:
    """The operands of a ``conditional`` call that can become its value: the THEN values and the ELSE of a CASE, the
    first argument of NULLIF, every argument of COALESCE / GREATEST / LEAST."""
    head = scalar_head(e.head)[0]
    if head == "CASE":
        return list(e.args[1::2]) + [e.args[-1]] if e.args else []
    return list(e.args[:1]) if head == "NULLIF" else list(e.args)


def is_string_build(e: Any) -> bool:
    """True for a node that builds a string: a call whose ``SCALARS`` result is ``string`` or ``||``."""
    if isinstance(e, ColumnExpr) and e.kind == Kind.BINARY:
        return e.head == "||"
    s = scalar_head(e.head) if isinstance(e, ColumnExpr) and e.kind == Kind.CALL else None
    return s is not None and s[1].result == "string"


def _str_arg(fn: str, what: str, v: Any) -> ColumnExpr:
    """A string literal argument (or NULL) of a string function."""
    e = _operand(v)
    if e.kind != Kind.LITERAL or e.as_type is not None:
        raise NotImplementedError(f"{fn}: {what} must be a string literal, got {e}")
    if e.value is not None and not isinstance(e.value, str):
        raise ValueError(f"{fn}: {what} must be a string literal or NULL, got {e.value!r}")
    return e


def case_string_results(e: Any) -> Optional[List[str]]:
    """The distinct string literals (in order of appearance) of a CASE / IF / IIF / NULLIF whose every result is a
    string literal or NULL, with at least one string; None for any other node."""
    s = scalar_head(e.head) if isinstance(e, ColumnExpr) and e.kind == Kind.CALL else None
    if s is None or s[1].result != "case":
        return None
    out: List[str] = []
    for r in result_args(e):
        r = _operand(r)
        if r.kind != Kind.LITERAL or r.as_type is not None or not (r.value is None or isinstance(r.value, str)):
            return None
        if r.value is not None and r.value not in out:
            out.append(r.value)
    return out if out else None


def _check_results(e: ColumnExpr) -> ColumnExpr:
    lits = [r for r in result_args(e) if r.kind == Kind.LITERAL and r.value is not None]
    if any(isinstance(r.value, str) for r in lits) and not all(isinstance(r.value, str) for r in lits):
        raise ValueError(f"{e.head} mixes string and numeric results: {e}")
    return e


def column_mentions(column: Any) -> Iterator[str]:
    """Names of the columns an expression reads."""
    if isinstance(column, ColumnExpr):
        if column.kind == Kind.NAMED:
            yield column.head
        for a in _children(column):
            yield from column_mentions(a)


class functions:
    """``f = fugue_b200.column.functions`` plays the role of ``import fugue.column.functions as f``."""

    @staticmethod
    def coalesce(*args: Any) -> ColumnExpr:
        return _call("COALESCE", *args)

    @staticmethod
    def case(branches: Sequence[Tuple[Any, Any]], else_: Any = None) -> ColumnExpr:
        """SQL ``CASE WHEN cond THEN value ... ELSE else_ END``: the value of the first branch whose condition is
        TRUE (NULL and FALSE fall through), else ``else_`` (NULL if not given).  The result is float64 if any branch
        is a float, bool if all are bool or NULL, else int64; string literals (and NULL) give a string column."""
        branches = list(branches)
        if not branches:
            raise ValueError("CASE needs at least one WHEN branch")
        args: List[Any] = []
        for b in branches:
            if not isinstance(b, tuple) or len(b) != 2:
                raise ValueError(f"a CASE branch is a (condition, value) pair, got {b!r}")
            args += list(b)
        return _check_results(_call("CASE", *args, else_))

    @staticmethod
    def nullif(a: Any, b: Any) -> ColumnExpr:
        """SQL ``NULLIF(a, b)``: NULL where ``a = b`` is TRUE, else ``a``."""
        return _call("NULLIF", a, b)

    @staticmethod
    def abs(c: Any) -> ColumnExpr:  # noqa: A003
        """``|c|``; an integer wraps at INT64_MIN as unary ``-`` does."""
        return _call("ABS", c)

    @staticmethod
    def floor(c: Any) -> ColumnExpr:
        return _call("FLOOR", c)

    @staticmethod
    def ceil(c: Any) -> ColumnExpr:
        return _call("CEIL", c)

    @staticmethod
    def round(c: Any, d: Any = 0) -> ColumnExpr:  # noqa: A003
        """SQL ``ROUND(c, d)``: to ``d`` decimal digits (an int literal in [-18, 18]), half away from zero."""
        return _call("ROUND", c, round_digits(d))

    @staticmethod
    def sqrt(c: Any) -> ColumnExpr:
        return _call("SQRT", c)

    @staticmethod
    def exp(c: Any) -> ColumnExpr:
        return _call("EXP", c)

    @staticmethod
    def ln(c: Any) -> ColumnExpr:
        return _call("LN", c)

    @staticmethod
    def log10(c: Any) -> ColumnExpr:
        return _call("LOG10", c)

    @staticmethod
    def power(a: Any, b: Any) -> ColumnExpr:
        return _call("POWER", a, b)

    @staticmethod
    def greatest(*args: Any) -> ColumnExpr:
        """The largest non-NULL argument (NULL only if all are NULL); floats in the order of aggregate MAX."""
        return _call("GREATEST", *args)

    @staticmethod
    def least(*args: Any) -> ColumnExpr:
        """The smallest non-NULL argument (NULL only if all are NULL); floats in the order of aggregate MIN."""
        return _call("LEAST", *args)

    @staticmethod
    def length(c: Any) -> ColumnExpr:
        """SQL ``LENGTH(c)``: the number of characters (code points) of a string, int64."""
        return _call("LENGTH", col(c))

    @staticmethod
    def upper(c: Any) -> ColumnExpr:
        """SQL ``UPPER(c)``: every code point by its simple (one to one) Unicode upper-case mapping."""
        return _call("UPPER", col(c))

    @staticmethod
    def lower(c: Any) -> ColumnExpr:
        """SQL ``LOWER(c)``: every code point by its simple (one to one) Unicode lower-case mapping."""
        return _call("LOWER", col(c))

    @staticmethod
    def substr(c: Any, start: Any, length: Any = None) -> ColumnExpr:
        """SQLite ``SUBSTR(c, start[, length])`` in code points: 1-based; a negative start counts from the end;
        a negative length takes the code points before start.  ``start`` / ``length`` are int literals; NULL
        (``null()``) gives NULL, and ``length=None`` means no length."""
        return _call("SUBSTR", col(c), start, *([] if length is None else [length]))

    @staticmethod
    def trim(c: Any, chars: Any = None) -> ColumnExpr:
        """SQLite ``TRIM(c[, chars])``: removes the code points of ``chars`` (default: the space U+0020 only)
        from both ends."""
        return _call("TRIM", col(c), *([] if chars is None else [chars]))

    @staticmethod
    def ltrim(c: Any, chars: Any = None) -> ColumnExpr:
        return _call("LTRIM", col(c), *([] if chars is None else [chars]))

    @staticmethod
    def rtrim(c: Any, chars: Any = None) -> ColumnExpr:
        return _call("RTRIM", col(c), *([] if chars is None else [chars]))

    @staticmethod
    def replace(c: Any, from_: Any, to: Any) -> ColumnExpr:
        """SQLite ``REPLACE(c, from_, to)``: every non-overlapping ``from_``, left to right, by ``to``; an empty
        ``from_`` leaves ``c`` unchanged."""
        return _call("REPLACE", col(c), from_, to)

    @staticmethod
    def regexp_matches(c: Any, pattern: Any) -> ColumnExpr:
        """DuckDB ``REGEXP_MATCHES(c, pattern)``: whether the regular expression matches somewhere in the string
        (RE2 semantics, the subset of ``fugue_b200.regex``).  ``pattern`` is a string literal; NULL gives NULL."""
        from . import regex

        p = _str_arg("REGEXP_MATCHES", "pattern", pattern)
        if p.value is not None:
            regex.parse(p.value)
        return _call("REGEXP_MATCHES", col(c), p)

    @staticmethod
    def regexp_full_match(c: Any, pattern: Any) -> ColumnExpr:
        """DuckDB ``REGEXP_FULL_MATCH(c, pattern)``: whether the regular expression matches the whole string."""
        from . import regex

        p = _str_arg("REGEXP_FULL_MATCH", "pattern", pattern)
        if p.value is not None:
            regex.parse(p.value)
        return _call("REGEXP_FULL_MATCH", col(c), p)

    @staticmethod
    def regexp_extract(c: Any, pattern: Any, group: Any = 0) -> ColumnExpr:
        """DuckDB ``REGEXP_EXTRACT(c, pattern[, group])``: the text of group ``group`` (0, the default: the whole
        match) of the leftmost match; '' when nothing matches or the group took no part.  A group above the
        pattern's group count is a ValueError."""
        from . import regex

        _, (s, p, g) = check_call("REGEXP_EXTRACT", [col(c), pattern, group])
        if p.value is not None:
            regex.parse(p.value)
            if g.value is not None:
                regex.check_group(p.value, g.value)
        return ColumnExpr(Kind.CALL, "REGEXP_EXTRACT", [s, p] + ([] if g.value == 0 else [g]))

    @staticmethod
    def regexp_replace(c: Any, pattern: Any, rewrite: Any, options: Any = None) -> ColumnExpr:
        """DuckDB ``REGEXP_REPLACE(c, pattern, rewrite[, options])``: the first match replaced by ``rewrite``, or
        every non-overlapping match with ``options='g'``.  In ``rewrite``, ``\\0`` .. ``\\9`` are groups and
        ``\\\\`` is a backslash."""
        from . import regex

        e = _call("REGEXP_REPLACE", col(c), pattern, rewrite, *([] if options is None else [options]))
        p, r, o = e.args[1], e.args[2], e.args[3] if len(e.args) > 3 else None
        if o is not None and o.value is not None:
            regex.replace_options(o.value)
        if p.value is not None:
            regex.parse(p.value)
            if r.value is not None:
                regex.rewrite_tokens(p.value, r.value)
        return e

    @staticmethod
    def concat(*parts: Any) -> ColumnExpr:
        """SQLite ``CONCAT(a, ...)``: the parts joined; NULL parts are skipped (``CONCAT(NULL)`` is '')."""
        return _call("CONCAT", *parts)

    @staticmethod
    def concat_strict(*parts: Any) -> ColumnExpr:
        """SQL ``a || b || ...`` (left-nested): the parts joined, NULL if any part is NULL."""
        if len(parts) < 2:
            raise ValueError("|| needs at least two operands")
        e = _operand(parts[0])
        for x in parts[1:]:
            e = binary("||", e, x)
        return e

    @staticmethod
    def extract(field: str, c: Any) -> ColumnExpr:
        """SQL ``EXTRACT(field FROM c)`` of a date or UTC timestamp (proleptic Gregorian, floor semantics before
        1970): ``year month day hour minute second`` (whole second 0-59) ``quarter dow`` (0 = Sunday) ``isodow``
        (1 = Monday ... 7) ``doy week`` (ISO 8601) ``isoyear``, int64; ``epoch``: float64 seconds since 1970-01-01."""
        field = _time_word("EXTRACT", "field", field, TIME_FIELDS + ("epoch",))
        return ColumnExpr(Kind.CALL, "EXTRACT", [_operand(c)], {"field": field})

    date_part = extract

    @staticmethod
    def date_trunc(part: str, c: Any) -> ColumnExpr:
        """SQL ``DATE_TRUNC(part, c)``: the start of the ``year quarter month week`` (Monday) ``day hour minute
        second`` that ``c`` lies in; keeps the type of ``c`` (a date stays a date)."""
        return ColumnExpr(Kind.CALL, "DATE_TRUNC", [_operand(c)], {"part": _time_word("DATE_TRUNC", "part", part, TIME_PARTS)})

    @staticmethod
    def datediff(part: str, a: Any, b: Any) -> ColumnExpr:
        """DuckDB's ``DATEDIFF(part, a, b)``: the number of ``part`` boundaries crossed from ``a`` to ``b`` (int64)."""
        return ColumnExpr(Kind.CALL, "DATEDIFF", [_operand(a), _operand(b)],
                          {"part": _time_word("DATEDIFF", "part", part, TIME_PARTS)})

    @staticmethod
    def add_months(c: Any, n: Any) -> ColumnExpr:
        """``c + n`` calendar months (``n`` an int or an int64 expression): the day is clamped to the last day of the
        target month (Jan 31 + 1 month = Feb 28 / 29), the time of day kept; Postgres, DuckDB, ``pandas.DateOffset``."""
        if isinstance(n, bool) or (not isinstance(n, (int, ColumnExpr))):
            raise ValueError(f"ADD_MONTHS: n must be an int or an integer expression, got {n!r}")
        return _call("ADD_MONTHS", c, n)

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
    def var_samp(c: Any) -> ColumnExpr:
        """Sample variance M2 / (m - 1) of the m non-NULL values (float64; NULL when m < 2)."""
        return agg("VAR_SAMP", c)

    variance = var_samp

    @staticmethod
    def var_pop(c: Any) -> ColumnExpr:
        """Population variance M2 / m of the m non-NULL values (float64; NULL when m = 0)."""
        return agg("VAR_POP", c)

    @staticmethod
    def stddev_samp(c: Any) -> ColumnExpr:
        """sqrt(VAR_SAMP): pandas ``std()`` (ddof = 1)."""
        return agg("STDDEV_SAMP", c)

    stddev = stddev_samp

    @staticmethod
    def stddev_pop(c: Any) -> ColumnExpr:
        """sqrt(VAR_POP): pandas ``std(ddof=0)``."""
        return agg("STDDEV_POP", c)

    # ---- shape statistics (DESIGN §7m) of the m non-NULL values, from their central sums Mk = sum of (x - mean)^k.
    # NaN and +-inf are values: one makes the result NaN.  A constant column gives 0.
    @staticmethod
    def skewness(c: Any) -> ColumnExpr:
        """Bias-corrected skewness G1 = m sqrt(m - 1) / (m - 2) * M3 / M2^1.5: pandas ``skew()`` (float64; NULL when
        m < 3)."""
        return agg("SKEWNESS", c)

    skew = skewness

    @staticmethod
    def skewness_pop(c: Any) -> ColumnExpr:
        """Population skewness g1 = sqrt(m) * M3 / M2^1.5 (float64; NULL when m = 0)."""
        return agg("SKEWNESS_POP", c)

    @staticmethod
    def kurtosis(c: Any) -> ColumnExpr:
        """Bias-corrected excess kurtosis G2 = m (m + 1) (m - 1) M4 / ((m - 2)(m - 3) M2^2) - 3 (m - 1)^2 /
        ((m - 2)(m - 3)): pandas ``kurt()`` (float64; NULL when m < 4)."""
        return agg("KURTOSIS", c)

    kurt = kurtosis

    @staticmethod
    def kurtosis_pop(c: Any) -> ColumnExpr:
        """Population excess kurtosis g2 = m M4 / M2^2 - 3: DuckDB ``kurtosis_pop`` (float64; NULL when m = 0)."""
        return agg("KURTOSIS_POP", c)

    # ---- two-argument aggregates (SQL:2003 binary set functions, DESIGN §7k).  Only the rows where both
    # arguments are non-NULL take part; m is their number.  NaN and +-inf are values, not NULL.
    @staticmethod
    def corr(a: Any, b: Any) -> ColumnExpr:
        """Pearson's correlation Sab / sqrt(Saa Sbb), clamped to [-1, 1] (float64; NULL when m = 0 or either
        argument is constant over the pair rows)."""
        return _bivariate("CORR", a, b)

    @staticmethod
    def covar_pop(a: Any, b: Any) -> ColumnExpr:
        """Population covariance Sab / m (float64; NULL when m = 0)."""
        return _bivariate("COVAR_POP", a, b)

    @staticmethod
    def covar_samp(a: Any, b: Any) -> ColumnExpr:
        """Sample covariance Sab / (m - 1): pandas ``cov()`` (float64; NULL when m < 2)."""
        return _bivariate("COVAR_SAMP", a, b)

    @staticmethod
    def regr_count(y: Any, x: Any) -> ColumnExpr:
        """m, the number of rows where both are non-NULL (int64, never NULL)."""
        return _bivariate("REGR_COUNT", y, x)

    @staticmethod
    def regr_avgx(y: Any, x: Any) -> ColumnExpr:
        """The mean of x over the pair rows (float64; NULL when m = 0)."""
        return _bivariate("REGR_AVGX", y, x)

    @staticmethod
    def regr_avgy(y: Any, x: Any) -> ColumnExpr:
        """The mean of y over the pair rows (float64; NULL when m = 0)."""
        return _bivariate("REGR_AVGY", y, x)

    @staticmethod
    def regr_sxx(y: Any, x: Any) -> ColumnExpr:
        """Sxx = sum of (x - mean x)^2 over the pair rows (float64; NULL when m = 0)."""
        return _bivariate("REGR_SXX", y, x)

    @staticmethod
    def regr_syy(y: Any, x: Any) -> ColumnExpr:
        """Syy = sum of (y - mean y)^2 over the pair rows (float64; NULL when m = 0)."""
        return _bivariate("REGR_SYY", y, x)

    @staticmethod
    def regr_sxy(y: Any, x: Any) -> ColumnExpr:
        """Sxy = sum of (x - mean x)(y - mean y) over the pair rows (float64; NULL when m = 0)."""
        return _bivariate("REGR_SXY", y, x)

    @staticmethod
    def regr_slope(y: Any, x: Any) -> ColumnExpr:
        """The least-squares slope Sxy / Sxx of y on x (float64; NULL when m = 0 or Sxx = 0)."""
        return _bivariate("REGR_SLOPE", y, x)

    @staticmethod
    def regr_intercept(y: Any, x: Any) -> ColumnExpr:
        """The least-squares intercept mean y - slope * mean x (float64; NULL when m = 0 or Sxx = 0)."""
        return _bivariate("REGR_INTERCEPT", y, x)

    @staticmethod
    def regr_r2(y: Any, x: Any) -> ColumnExpr:
        """The coefficient of determination: 1 when Syy = 0, else Sxy^2 / (Sxx Syy) clamped to [0, 1] (float64;
        NULL when m = 0 or Sxx = 0)."""
        return _bivariate("REGR_R2", y, x)

    @staticmethod
    def percentile_cont(c: Any, q: Any) -> ColumnExpr:
        """The q-quantile of the non-NULL values, interpolated linearly between the two nearest (float64)."""
        return _percentile("PERCENTILE_CONT", c, q)

    @staticmethod
    def percentile_disc(c: Any, q: Any) -> ColumnExpr:
        """The first value (in ascending order) whose cumulative distribution reaches q; keeps the type."""
        return _percentile("PERCENTILE_DISC", c, q)

    @staticmethod
    def median(c: Any) -> ColumnExpr:
        """``percentile_cont(c, 0.5)``: the same node."""
        return _percentile("PERCENTILE_CONT", c, 0.5)

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

    @staticmethod
    def ntile(n: int) -> ColumnExpr:
        """SQL NTILE: the bucket 1..n of the row in partition order, bucket sizes differing by at most one, the
        larger buckets first (1..N when the partition has N < n rows)."""
        return ColumnExpr(Kind.WINDOW, "NTILE", [], {"n": _nth("NTILE", n)})

    @staticmethod
    def percent_rank() -> ColumnExpr:
        """SQL PERCENT_RANK: (RANK - 1) / (partition rows - 1), 0 in a partition of one row (float64)."""
        return ColumnExpr(Kind.WINDOW, "PERCENT_RANK")

    @staticmethod
    def cume_dist() -> ColumnExpr:
        """SQL CUME_DIST: the rows up to and including the current row's last peer over the partition's rows."""
        return ColumnExpr(Kind.WINDOW, "CUME_DIST")

    @staticmethod
    def first_value(c: Any) -> ColumnExpr:
        """SQL FIRST_VALUE: ``c`` at the first row of the frame, NULL included (FIRST skips NULLs); NULL for an empty
        frame.  The frame is the whole partition unless ``over()`` gives one."""
        return _value_fn("FIRST_VALUE", c, {})

    @staticmethod
    def last_value(c: Any) -> ColumnExpr:
        """SQL LAST_VALUE: ``c`` at the last row of the frame, NULL included; NULL for an empty frame."""
        return _value_fn("LAST_VALUE", c, {})

    @staticmethod
    def ewm_mean(c: Any, com: Any = None, span: Any = None, halflife: Any = None, alpha: Any = None, *,
                 adjust: bool = True, ignore_na: bool = False, min_periods: int = 0, times: bool = False) -> ColumnExpr:
        """pandas' ``ewm(...).mean()`` over the logical partition in presort (or ORDER BY) order, as a window function
        (float64).  Exactly one of ``com``, ``span``, ``halflife`` and ``alpha`` gives the decay; ``times=True`` decays
        by 0.5^(dt / halflife) over the single order column (ascending, no NULLs).  An observation is a non-NULL,
        non-NaN value of ``c`` (an integer or float column); NULL before the first observation and while fewer than
        ``min_periods`` observations are in, and a row without a value repeats the last result.  No frame."""
        return _ewm_fn("EWM_MEAN", c, dict(com=com, span=span, halflife=halflife, alpha=alpha), adjust, ignore_na,
                       min_periods, times)

    @staticmethod
    def ewm_var(c: Any, com: Any = None, span: Any = None, halflife: Any = None, alpha: Any = None, *,
                adjust: bool = True, ignore_na: bool = False, min_periods: int = 0, bias: bool = False,
                times: bool = False) -> ColumnExpr:
        """pandas' ``ewm(...).var(bias=bias)``: the weighted variance C / W about the weighted mean, times W^2 / (W^2 -
        W2) unless ``bias`` (NULL below two observations).  Options as :meth:`ewm_mean`; time decay is not supported."""
        return _ewm_fn("EWM_VAR", c, dict(com=com, span=span, halflife=halflife, alpha=alpha), adjust, ignore_na,
                       min_periods, times, bias)

    @staticmethod
    def ewm_std(c: Any, com: Any = None, span: Any = None, halflife: Any = None, alpha: Any = None, *,
                adjust: bool = True, ignore_na: bool = False, min_periods: int = 0, bias: bool = False,
                times: bool = False) -> ColumnExpr:
        """pandas' ``ewm(...).std(bias=bias)``: the square root of :meth:`ewm_var`."""
        return _ewm_fn("EWM_STD", c, dict(com=com, span=span, halflife=halflife, alpha=alpha), adjust, ignore_na,
                       min_periods, times, bias)

    @staticmethod
    def nth_value(c: Any, n: int) -> ColumnExpr:
        """SQL NTH_VALUE: ``c`` at the frame's ``n``-th row (``n >= 1``), NULL included; NULL when the frame has fewer
        than ``n`` rows."""
        return _value_fn("NTH_VALUE", c, {"n": _nth("NTH_VALUE", n)})


def _time_word(fn: str, what: str, word: Any, known: Tuple[str, ...]) -> str:
    if not isinstance(word, str) or word.lower() not in known:
        raise ValueError(f"{fn}: unknown {what} {word!r}; one of {', '.join(known)}")
    return word.lower()


for _field in ("year", "month", "day", "hour", "minute", "second", "quarter"):
    setattr(functions, _field, staticmethod(lambda c, _f=_field: functions.extract(_f, c)))
for _name, _field in (("dayofweek", "dow"), ("dayofyear", "doy"), ("week", "week")):
    setattr(functions, _name, staticmethod(lambda c, _f=_field: functions.extract(_f, c)))


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
                               if self._role(c) in ("simple", "func") and not has_window(c)]

    @staticmethod
    def _role(c: ColumnExpr) -> str:
        if c.kind == Kind.LITERAL:
            return "literal"
        if c.kind in (Kind.NAMED, Kind.WILDCARD):
            return "simple"
        return "agg" if is_agg(c) or window_reads_agg(c) else "func"

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
_SQL_OF_OP = {"&": " AND ", "|": " OR ", "==": "=", "||": " || "}


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
    elif k == Kind.AGG and expr.head in PERCENTILES:
        body = _within_group(expr, lambda x: to_sql(x, enable_cast))
    elif k == Kind.CALL and expr.head == "LIKE":
        body = to_sql(expr.args[0], enable_cast, True) + " LIKE " + to_sql(expr.args[1], enable_cast)
        if len(expr.args) > 2:
            body += " ESCAPE " + to_sql(expr.args[2], enable_cast)
        if nested:
            body = "(" + body + ")"
    elif k == Kind.CALL and expr.head.upper() in SCALARS and SCALARS[expr.head.upper()].family == "regex":
        # the SQL parser reads a regular expression's string literals as written: only '' is a quote
        parts = [to_sql(expr.args[0], enable_cast)] + [
            "'" + x.value.replace("'", "''") + "'" if x.kind == Kind.LITERAL and isinstance(x.value, str)
            and x.as_type is None else to_sql(_operand(x), enable_cast) for x in expr.args[1:]]
        body = f"{expr.head.upper()}({','.join(parts)})"
    elif k == Kind.CALL and expr.head.upper() in ("EXTRACT", "DATE_TRUNC", "DATEDIFF") and \
            isinstance(expr.kwargs.get("field" if expr.head.upper() == "EXTRACT" else "part"), str):
        inner = ", ".join(to_sql(_operand(x), enable_cast) for x in expr.args)
        body = f"EXTRACT({expr.kwargs['field']} FROM {inner})" if expr.head.upper() == "EXTRACT" else \
            f"{expr.head.upper()}('{expr.kwargs['part']}', {inner})"
    elif k == Kind.CALL and expr.head.upper() == "CASE" and len(expr.args) % 2 == 1:
        a = expr.args
        body = "CASE" + "".join(f" WHEN {to_sql(_operand(a[i]), enable_cast)} THEN {to_sql(_operand(a[i + 1]), enable_cast)}"
                                for i in range(0, len(a) - 1, 2)) + f" ELSE {to_sql(_operand(a[-1]), enable_cast)} END"
    elif k == Kind.BINARY:
        if expr.head not in BOOL_OPS and expr.head not in ARITH_OPS and expr.head != "||":
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
