"""Compile column expressions (``fugue_b200.column``) into programs for the device evaluator.

``project`` / ``filter_table`` are what ``B200ExecutionEngine.select / filter / assign`` run on: the
reference generates SQL text for these trees and lets qpd/pandas evaluate it operator by operator
(fugue/execution/execution_engine.py:736-887, fugue/column/sql.py:275-347); here a whole SELECT list is
one register-machine program and one pass over HBM (``fb_eval_expr``, fugue_b200/csrc/fb_expr.cu).

Typing rules (the reference leaves them to the SQL engine; these are the pandas/qpd ones):
``+ - *`` on integers -> int64, with any float -> float64; ``/`` -> float64 (true division);
comparisons / ``& | ~`` / ``IS NULL`` -> bool with SQL three-valued logic; an explicit ``cast`` wins.
String columns are dictionary encoded: they can be passed through, tested for NULL and compared
(``==`` / ``!=``) with a string literal.  ``CAST(x AS STRING)`` of a number, bool, date or timestamp formats every
distinct value once (``strings.format_values``, K14) into a dictionary column; inside an expression it becomes a
temporary column of a wider table first (``_string_casts``), which every string consumer takes as a string column.
``LIKE`` and ``LENGTH`` of a string column are computed once per dictionary entry (``strings.py``) and
read per row through the entry's code (``FB_X_LOOKUP``), inside the same program.
``CASE`` runs without branching (every branch on every row, ``FB_X_SEL`` picks); its class, and that of
``GREATEST`` / ``LEAST``, is COALESCE's rule.  ``%`` and ``ABS FLOOR CEIL ROUND`` keep the operand's class
(int64 or float64), ``SQRT EXP LN LOG10 POWER`` are float64.  A CASE whose results are string literals is a
whole output column only: ``project`` compiles it to int32 codes into a dictionary of those literals.
A string-building expression over one string column (``UPPER LOWER SUBSTR TRIM LTRIM RTRIM REPLACE CONCAT ||``)
is evaluated over the dictionary (``strings.evaluate``); per row it is the code (``FB_X_MOV``) mapped to the
result's code in a new dictionary (``FB_X_LOOKUP``).  It is a whole output column (``project``), or the
operand of ``==`` / ``!=`` with a string literal, of ``IS [NOT] NULL``, of ``LIKE`` and of ``LENGTH``.
Dates and timestamps are int64 counts of their Arrow unit.  A temporal literal (``DATE '..'``, ``TIMESTAMP '..'``, an
interval) is rescaled on the host to the unit of the temporal operand it meets and becomes a plain immediate; two
temporal columns meet as their raw integers, and the unit-correct form is an explicit ``CAST`` between temporal types
(``FB_X_MULSAT_I`` / ``FB_X_FLOORDIV_I``).  ``EXTRACT DATE_TRUNC DATEDIFF ADD_MONTHS`` are the ``FB_X_TS_*`` ops.
A ``CAST`` of a string column, or of a string-building expression, to a number, bool, date or timestamp is Arrow's
``cast(safe=False)`` of the entry: every entry is parsed once (``strings.parse_table``, K13) and each row reads its
entry's value (``FB_X_LOOKUP``); the result has the target's class and, for a date or timestamp, its unit.  A string
that does not parse raises ValueError when a valid row refers to it.  A cast string literal is cast on the host.
"""
import datetime
import struct
from typing import Any, Dict, List, Optional, Sequence, Tuple

import pyarrow as pa
import torch

from . import kernels as K
from . import strings as ST
from .column import (REGEX_PREDICATES, TEMPORAL_LITERALS, TIME_FIELDS, TIME_PARTS, ColumnExpr, Kind, Scalar,
                     _children, case_string_results, check_call, col as _col, is_string_build, lit as _lit, result_args, round_digits,
                     scalar_head)
from .schema import Schema
from .table import B200Table, _storage_dtype, expr_type


def _is_str(tp: Optional[pa.DataType]) -> bool:
    return tp is not None and (pa.types.is_string(tp) or pa.types.is_large_string(tp))


def _cls_of(tp: pa.DataType) -> str:
    if pa.types.is_boolean(tp):
        return "b"
    if pa.types.is_floating(tp):
        return "f"
    if _is_str(tp):
        return "s"
    return "i"  # integers, dates, timestamps: int64 arithmetic


def _f64_bits(v: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(v)))[0]


_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1
_EPOCH = datetime.datetime(1970, 1, 1)
_US = datetime.timedelta(microseconds=1)
# units of one microsecond as a fraction (numerator, denominator), by unit code (kernels.TU_*)
_PER_US = {K.TU_DAY: (1, 86_400_000_000), K.TU_S: (1, 1_000_000), K.TU_MS: (1, 1000), K.TU_US: (1, 1), K.TU_NS: (1000, 1)}
_UNIT_CODE = {"s": K.TU_S, "ms": K.TU_MS, "us": K.TU_US, "ns": K.TU_NS}


def time_unit(tp: Optional[pa.DataType]) -> Optional[Tuple[str, int]]:
    """``("point" | "span", unit code)`` of a date / timestamp / duration type, None for every other type."""
    if tp is None:
        return None
    if pa.types.is_date32(tp):
        return "point", K.TU_DAY
    if pa.types.is_date64(tp):
        return "point", K.TU_MS
    if pa.types.is_timestamp(tp):
        return "point", _UNIT_CODE[tp.unit]
    if pa.types.is_duration(tp):
        return "span", _UNIT_CODE[tp.unit]
    return None


def _literal_us(v: Any) -> int:
    """A temporal literal as exact microseconds (since the epoch for a date or timestamp; a date is its midnight)."""
    if isinstance(v, datetime.timedelta):
        return v // _US
    if not isinstance(v, datetime.datetime):
        v = datetime.datetime(v.year, v.month, v.day)
    return (v - _EPOCH) // _US


def _natural_type(v: Any) -> pa.DataType:
    return pa.duration("us") if isinstance(v, datetime.timedelta) else \
        pa.timestamp("us") if isinstance(v, datetime.datetime) else pa.date32()


def _is_temporal_literal(e: Any) -> bool:
    return isinstance(e, ColumnExpr) and e.kind == Kind.LITERAL and e.as_type is None and \
        isinstance(e.value, TEMPORAL_LITERALS)


def _in_unit(v: Any, unit: int) -> Tuple[int, bool]:
    """(floor of the literal in ``unit``, whether it is a whole number of them)."""
    num, den = _PER_US[unit]
    q, r = divmod(_literal_us(v) * num, den)
    return q, r == 0


def _const_predicate(x: ColumnExpr, truth: bool) -> ColumnExpr:
    """``truth`` where ``x`` is not NULL, NULL elsewhere (Kleene: TRUE OR NULL, FALSE AND NULL)."""
    return (x.not_null() | _lit(None)) if truth else (x.is_null() & _lit(None))


def string_literal_cast(e: ColumnExpr) -> ColumnExpr:
    """``CAST('text' AS tp)`` folded on the host by Arrow's cast: a literal of the value's class that keeps the cast
    (a date or timestamp is its count of the type's unit) and the alias.  ValueError when the text does not parse,
    NotImplementedError for a target the device does not parse to."""
    import pyarrow.compute as pc

    tp = e.as_type
    ST.parse_target(tp)
    try:
        v = pc.cast(pa.array([e.value], type=pa.string()), tp, safe=False)
    except (pa.ArrowInvalid, pa.ArrowNotImplementedError):
        raise ST.parse_error(e.value, tp) from None
    if pa.types.is_date32(tp):
        py: Any = v.view(pa.int32())[0].as_py()
    elif pa.types.is_date64(tp) or pa.types.is_timestamp(tp):
        py = v.view(pa.int64())[0].as_py()
    else:
        py = v[0].as_py()
    out = _lit(py).cast(tp)
    return out.alias(e.as_name) if e.as_name != "" else out


class _OutOfResources(Exception):
    pass


def _regex_pattern(e: ColumnExpr, fn: str) -> Optional[str]:
    """The pattern of REGEXP_MATCHES / REGEXP_FULL_MATCH (None: a NULL literal, so the result is NULL)."""
    p = e.args[1]
    if p.kind != Kind.LITERAL or p.as_type is not None or not (p.value is None or isinstance(p.value, str)):
        raise NotImplementedError(f"{fn} needs a string literal pattern: {e}")
    return p.value


def _like_pattern(e: ColumnExpr) -> Tuple[str, Optional[str]]:
    """The pattern and the escape character (None: none) of a LIKE."""
    if not all(a.kind == Kind.LITERAL and isinstance(a.value, str) for a in e.args[1:]):
        raise NotImplementedError(f"LIKE needs a string literal pattern: {e}")
    return e.args[1].value, (e.args[2].value if len(e.args) > 2 else None)


def _scalar(e: Any) -> Tuple[Optional[str], Optional[Scalar]]:
    """The canonical head and ``SCALARS`` entry of a call, (None, None) for any other node."""
    s = scalar_head(e.func) if isinstance(e, ColumnExpr) and e.kind == Kind.CALL else None
    return s if s is not None else (None, None)


def _canonical(e: ColumnExpr) -> ColumnExpr:
    """A call of a ``SCALARS`` function, its arguments checked (``check_call``), in its canonical spelling (no alias,
    no cast); NULLIF(a, b) as CASE WHEN a = b THEN NULL ELSE a END and MOD(a, b) as a % b."""
    head, args = check_call(e.func, e.args)
    if head == "NULLIF":
        return ColumnExpr(Kind.CALL, "CASE", [ColumnExpr(Kind.BINARY, "==", args), _lit(None), args[0]])
    if head == "MOD":
        return ColumnExpr(Kind.BINARY, "%", args)
    return ColumnExpr(Kind.CALL, head, args, e.kwargs)


def _coalesce_cls(cs: Sequence[str]) -> str:
    """COALESCE's result class: float64 if any is a float, bool if all are bool / NULL, else int64."""
    return "f" if "f" in cs else ("b" if "b" in cs and all(c in ("b", "n") for c in cs) else "i")


class _Program:
    """One ``fb_eval_expr`` launch.  Code generation for the accumulator machine: ``compile`` leaves the
    value of an expression in the accumulator; the right-hand side of an operator is used in place
    when it is a leaf (column / literal), otherwise the left value waits in a temporary."""

    _REVERSE = {"+": "+", "*": "*", "-": "r-", "/": "r/", "<": ">", "<=": ">=", ">": "<", ">=": "<=",
                "==": "==", "!=": "!=", "&": "&", "|": "|", "%": "r%", "**": "r**"}
    _OPS = {  # (int opcode, float opcode)
        "+": (K.X_ADD_I, K.X_ADD_F), "-": (K.X_SUB_I, K.X_SUB_F), "r-": (K.X_RSUB_I, K.X_RSUB_F),
        "*": (K.X_MUL_I, K.X_MUL_F), "/": (None, K.X_DIV_F), "r/": (None, K.X_RDIV_F),
        "<": (K.X_LT_I, K.X_LT_F), "<=": (K.X_LE_I, K.X_LE_F), ">": (K.X_GT_I, K.X_GT_F),
        ">=": (K.X_GE_I, K.X_GE_F), "==": (K.X_EQ_I, K.X_EQ_F), "!=": (K.X_NE_I, K.X_NE_F),
        "%": (K.X_MOD_I, K.X_MOD_F), "r%": (K.X_RMOD_I, K.X_RMOD_F),
        "**": (None, K.X_POW), "r**": (None, K.X_RPOW),  # "**" is POWER(a, b), only inside the compiler
    }
    _UNARY_FN = {"ABS": (K.X_ABS_I, K.X_ABS_F), "FLOOR": (None, K.X_FLOOR_F), "CEIL": (None, K.X_CEIL_F),
                 "ROUND": (K.X_ROUND_I, K.X_ROUND_F), "SQRT": (None, K.X_SQRT), "EXP": (None, K.X_EXP),
                 "LN": (None, K.X_LN), "LOG10": (None, K.X_LOG10)}

    def __init__(self, table: B200Table):
        self.t = table
        self.ins: List[Tuple[int, int, int, int, int]] = []
        self.cols: List[Any] = []          # table column indices / lookup-table keys, in load order
        self.tables: Dict[Any, Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}  # key -> per-entry table
        self.free = list(range(K.EXPR_NREGS - 1, -1, -1))
        self.outs: List[Tuple[torch.dtype, bool, int]] = []  # (dtype, want_valid, K8 type) per FB_X_OUT

    # -- resources
    def alloc(self) -> int:
        if not self.free:
            raise _OutOfResources("temporaries")
        return self.free.pop()

    def release(self, r: int) -> None:
        self.free.append(r)

    def emit(self, op: int, kind: int = K.XK_NONE, b: int = 0, flags: int = 0, imm: int = 0) -> None:
        if len(self.ins) >= K.EXPR_MAX_INS:
            raise _OutOfResources("instructions")
        self.ins.append((op, kind, b, flags, imm))

    def col_slot(self, ci: Any) -> int:
        if ci in self.cols:
            return self.cols.index(ci)
        if len(self.cols) >= K.EXPR_MAX_COLS:
            raise _OutOfResources("columns")
        self.cols.append(ci)
        return len(self.cols) - 1

    def output(self, dtype: torch.dtype, want_valid: bool, tp: Optional[int] = None) -> None:
        """``tp``: the K8 type of the output (default: the signed integer or float of ``dtype``)."""
        if len(self.outs) >= K.EXPR_MAX_OUTS:
            raise _OutOfResources("outputs")
        self.emit(K.X_OUT, K.XK_NONE, len(self.outs))
        self.outs.append((dtype, want_valid, K.expr_type_of(dtype) if tp is None else tp))

    def mark(self) -> Any:
        return (len(self.ins), list(self.cols), list(self.free), len(self.outs))

    def rollback(self, m: Any) -> None:
        del self.ins[m[0]:]
        self.cols, self.free = m[1], m[2]
        del self.outs[m[3]:]

    # -- leaves: usable directly as operand B.  Returns (kind, b, imm, cls, nullable) or None
    def _leaf(self, e: Any) -> Optional[Tuple[int, int, int, str, bool]]:
        if e.as_type is not None:
            return None
        if e.kind == Kind.NAMED:
            t = self.t
            if e.name not in t.schema:
                raise KeyError(f"column {e.name} is not in {t.schema}")
            ci = t.schema.index_of_key(e.name)
            cls = _cls_of(t.schema.types[ci])
            return (K.XK_COL, ci, 0, cls, t.valid[ci] is not None)  # b = table column, slot assigned on use
        if e.kind == Kind.LITERAL:
            v = e.value
            if v is None:
                return (K.XK_NULL, 0, 0, "n", True)
            if isinstance(v, bool):
                return (K.XK_IMM, 0, int(v), "b", False)
            if isinstance(v, int):
                return (K.XK_IMM, 0, v & ((1 << 64) - 1), "i", False)
            if isinstance(v, float):
                return (K.XK_IMM, 0, _f64_bits(v), "f", False)
            if isinstance(v, TEMPORAL_LITERALS):  # alone: in the unit of its own type (days / microseconds)
                q, _ = _in_unit(v, time_unit(_natural_type(v))[1])
                return (K.XK_IMM, 0, q & ((1 << 64) - 1), "i", False)
        return None

    def _emit_with(self, op: int, leaf: Tuple[int, int, int, str, bool], ctx: str, flags: int = 0) -> None:
        """``acc <- acc op leaf`` with the leaf converted to the context class ('i', 'f' or 'b')."""
        kind, b, imm, cls, _ = leaf
        if kind == K.XK_COL:
            b = self.col_slot(b)
            if ctx == "f" and cls != "f":
                flags |= K.XF_B_I2F
        elif kind == K.XK_IMM and ctx == "f" and cls != "f":
            v = imm - (1 << 64) if imm >= (1 << 63) else imm
            imm = _f64_bits(float(v))
        self.emit(op, kind, b, flags, imm)

    def _acc_to(self, cls: str, ctx: str) -> None:
        if cls == "n" or cls == ctx:
            return
        if ctx == "f":
            # peephole: the accumulator was just loaded from an integer leaf -> convert while loading
            if self.ins and self.ins[-1][0] == K.X_MOV and self.ins[-1][3] == 0:
                op, kind, b, _, imm = self.ins[-1]
                if kind == K.XK_COL:
                    self.ins[-1] = (op, kind, b, K.XF_B_I2F, imm)
                    return
                if kind == K.XK_IMM:
                    v = imm - (1 << 64) if imm >= (1 << 63) else imm
                    self.ins[-1] = (op, kind, b, 0, _f64_bits(float(v)))
                    return
            self.emit(K.X_I2F)
        elif ctx == "b":
            self.emit(K.X_TOBOOL_F if cls == "f" else K.X_TOBOOL_I)
        elif ctx == "i" and cls == "f":
            self.emit(K.X_F2I)

    # -- compilation: value ends up in the accumulator; returns (class, nullable)
    def compile(self, e: ColumnExpr, top: bool = False) -> Tuple[str, bool]:
        if e.as_type is not None and not _is_str(e.as_type):
            if e.kind == Kind.LITERAL and isinstance(e.value, str):
                return self.compile(string_literal_cast(e))
            if self._is_string_operand(e.cast(None)):
                return self._parse_cast(e)
        cls, nullable = self._node(e)
        if e.as_type is not None:
            want = _cls_of(e.as_type)
            if want == "s":
                if not top and cls != "s":
                    raise NotImplementedError(f"cast to str inside an expression (only on a whole column): {e}")
            elif cls == "s":
                raise NotImplementedError(f"cast of a string expression to {e.as_type}: {e}")
            elif cls != "n":
                self._temporal_cast(e)
                self._acc_to(cls, want)
                cls = want
        return cls, nullable

    # -- casts from strings
    def _is_string_operand(self, x: ColumnExpr) -> bool:
        """A string column or a string-building expression (what a cast can parse)."""
        if x.kind == Kind.NAMED:
            return x.as_type is None and x.name in self.t.schema and _is_str(self.t.schema[x.name].type)
        return is_string_build(x) and (x.as_type is None or _is_str(x.as_type))

    def _parse_cast(self, e: ColumnExpr) -> Tuple[str, bool]:
        """``CAST(s AS tp)``: the entry's code, then ``FB_X_LOOKUP`` into the dictionary's parse table.  Raises
        ValueError when a valid row refers to an entry that does not parse."""
        t, tp, x = self.t, e.as_type, e.cast(None)
        ST.parse_target(tp)  # NotImplementedError before anything runs for a target the device does not parse to
        if x.kind == Kind.NAMED:
            d = t.dictionaries[x.name]
            ci = t.schema.index_of_key(x.name)
            r = ST.parse_table(d, t.device, tp)
            ST.check_referenced(r, d, tp, t.columns[ci], t.valid[ci])
            key: Any = ("PARSE", x.name, tp)
            self.emit(K.X_MOV, K.XK_COL, self.col_slot(ci))
            row_null = t.valid[ci] is not None
        else:
            name, steps = ST.string_chain(x, t.dictionaries)
            src = ST.evaluate(t.dictionaries[name], t.device, steps)
            d, row_null = self.string_codes(x)
            r = ST.parse_table(d, t.device, tp)
            ci = t.schema.index_of_key(name)
            ST.check_referenced(r, d, tp, t.columns[ci], t.valid[ci], src.remap, src.remap_valid, src.null_code)
            key = ("PARSE", ("STR", name, steps), tp)
        values, valid = r.values, r.valid
        if len(d) == 0:  # every row is NULL: a one-entry table that is never read, for a real device pointer
            values = torch.zeros(1, dtype=torch.int64, device=t.device)
            valid = torch.zeros(1, dtype=torch.uint8, device=t.device)
        self.tables[key] = (values, valid)
        self.emit(K.X_LOOKUP, K.XK_COL, self.col_slot(key), 0, len(d))
        return _cls_of(tp), row_null or valid is not None

    # -- dates and timestamps
    def _ttype(self, e: Any) -> Optional[pa.DataType]:
        """The date / timestamp / duration type whose unit the value of ``e`` is counted in; None if it is not temporal
        (a temporal literal alone has none: it takes the unit of the operand it meets)."""
        if not isinstance(e, ColumnExpr):
            return None
        if e.as_type is not None:
            return e.as_type if time_unit(e.as_type) else None
        if e.kind == Kind.NAMED:
            tp = self.t.schema[e.name].type if e.name in self.t.schema else None
            return tp if time_unit(tp) else None
        if e.kind == Kind.BINARY and e.op in ("+", "-"):
            for x, d in ((e.left, e.right), (e.right, e.left)):
                if _is_temporal_literal(d) and isinstance(d.value, datetime.timedelta) and (e.op == "+" or d is e.right):
                    return self._ttype(x)
            return None
        s = _scalar(e)[1]
        if s is not None and s.result == "operand":
            return self._operand_type(e.args[0]) if e.args else None
        if s is not None and s.family == "conditional":
            for a in result_args(e):
                tp = self._ttype(a)
                if tp is not None:
                    return tp
        return None

    def _operand_type(self, e: Any) -> Optional[pa.DataType]:
        """``_ttype``, and for a temporal literal the type of the literal itself."""
        e = e if isinstance(e, ColumnExpr) else _lit(e)
        return _natural_type(e.value) if _is_temporal_literal(e) else self._ttype(e)

    def _temporal_cast(self, e: ColumnExpr) -> None:
        """``CAST`` between two date / timestamp types or two durations: the accumulator rescaled to the target's unit.
        To a finer unit the product saturates (it keeps its order against every value that fits); to a coarser one the
        division floors (``CAST(ts AS date)`` is the calendar day, also before 1970)."""
        dst, src = time_unit(e.as_type), time_unit(self._operand_type(e.cast(None)))
        if dst is None or src is None or dst[0] != src[0] or dst[1] == src[1]:
            return
        (n1, d1), (n2, d2) = _PER_US[src[1]], _PER_US[dst[1]]
        num, den = n2 * d1, d2 * n1  # target units per source unit
        if num >= den:
            self.emit(K.X_MULSAT_I, K.XK_IMM, 0, 0, num // den)
        else:
            self.emit(K.X_FLOORDIV_I, K.XK_IMM, 0, 0, den // num)

    def _literal_for(self, v: Any, tp: pa.DataType, what: Any) -> ColumnExpr:
        """A temporal literal as the int64 literal of its exact value in the unit of ``tp`` (clamped to int64)."""
        kind, unit = time_unit(tp)
        if (kind == "span") != isinstance(v, datetime.timedelta):
            raise ValueError(f"{_lit(v)} can't stand for a value of type {tp}: {what}")
        q, exact = _in_unit(v, unit)
        if not exact:
            raise ValueError(f"{_lit(v)} is not a whole number of the units of {tp}: {what}")
        return _lit(min(max(q, _I64_MIN), _I64_MAX))

    def _temporal_operands(self, e: ColumnExpr) -> ColumnExpr:  # noqa: C901
        """The node with its temporal literals replaced by int64 literals in the unit of the temporal operand they
        meet (comparison, ``+ -``, COALESCE, CASE result, GREATEST / LEAST), so that no device instruction is spent
        on them.  Two literals fold on the host."""
        if e.kind == Kind.BINARY and e.op in ("+", "-", "<", "<=", ">", ">=", "==", "!="):
            a, b = _folded(e.left), _folded(e.right)
            la, lb = _is_temporal_literal(a), _is_temporal_literal(b)
            if not (la or lb):
                return e
            if la and lb:
                return _fold(e.op, a.value, b.value, e)
            x, l, lit_left = (b, a, True) if la else (a, b, False)
            v = l.value
            tp = self._ttype(x)
            if tp is None:
                raise ValueError(f"{l} meets an operand that is not a date, timestamp or duration: {e}")
            kind, unit = time_unit(tp)
            span = isinstance(v, datetime.timedelta)
            if e.op in ("+", "-"):
                if e.op == "+" and not span:
                    raise ValueError(f"a date or timestamp can't be added to another: {e}")
                if span and e.op == "-" and lit_left and kind == "point":
                    raise ValueError(f"an interval minus a date or timestamp has no meaning: {e}")
                q, exact = _in_unit(v, unit)
                if not exact:
                    raise ValueError(f"{l} is not a whole number of the units of {tp} (cast the operand first): {e}")
                n = _lit(min(max(q, _I64_MIN), _I64_MAX))
                return ColumnExpr(Kind.BINARY, e.op, [n, x] if lit_left else [x, n])
            if span != (kind == "span"):
                raise ValueError(f"{l} can't be compared with a value of type {tp}: {e}")
            op = _Program._REVERSE[e.op] if lit_left else e.op  # x op literal
            q, exact = _in_unit(v, unit)
            if q > _I64_MAX or q < _I64_MIN:  # beyond every value of the unit
                return _const_predicate(x, op in (("<", "<=", "!=") if q > _I64_MAX else (">", ">=", "!=")))
            if not exact:
                if op in ("==", "!="):
                    return _const_predicate(x, op == "!=")
                if op in (">=", "<"):  # x >= v <=> x >= ceil(v); x < v <=> x < ceil(v)
                    if q == _I64_MAX:
                        return _const_predicate(x, op == "<")
                    q += 1
            return ColumnExpr(Kind.BINARY, op, [x, _lit(q)])
        if e.kind == Kind.CALL and _scalar(e)[1].family == "conditional":
            args = list(e.args)
            n = len(args)
            results = [i for i in range(n) if e.head != "CASE" or i % 2 == 1 or i == n - 1]
            if not any(_is_temporal_literal(args[i]) for i in results):
                return e
            tp = self._ttype(e)
            if tp is None:
                kinds = {isinstance(args[i].value, datetime.timedelta) for i in results if _is_temporal_literal(args[i])}
                if len(kinds) > 1:
                    raise ValueError(f"{e.func} mixes points in time and intervals: {e}")
                tp = pa.duration("us") if True in kinds else pa.timestamp("us")  # literals only
            for i in results:
                if _is_temporal_literal(args[i]):
                    args[i] = self._literal_for(args[i].value, tp, e)
            return ColumnExpr(Kind.CALL, e.head, args, e.kwargs)
        return e

    def _calendar_unit(self, e: ColumnExpr, a: Any) -> int:
        """The unit of a calendar function's date / timestamp operand; raises for what the device has no calendar for."""
        tp = self._operand_type(a)
        if tp is None:
            at = a.infer_type(self.t.schema) if isinstance(a, ColumnExpr) else None
            if at is not None and (pa.types.is_time(at) or pa.types.is_duration(at)):
                raise NotImplementedError(f"{e.func} of a {at} value: {e}")
            raise ValueError(f"{e.func} needs a date or timestamp operand, got {a}: {e}")
        if time_unit(tp)[0] != "point":
            raise NotImplementedError(f"{e.func} of a {tp} value: {e}")
        if pa.types.is_timestamp(tp) and tp.tz is not None and tp.tz.upper() != "UTC":
            raise NotImplementedError(f"{e.func} of a timestamp in time zone {tp.tz} (only UTC; there is no time-zone "
                                      f"database on the device): {e}")
        return time_unit(tp)[1]

    def _temporal_function(self, e: ColumnExpr, fn: str) -> Tuple[str, bool]:
        args = e.args
        word = e.kwargs.get("field" if fn == "EXTRACT" else "part")
        if fn != "ADD_MONTHS":
            known = TIME_FIELDS + ("epoch",) if fn == "EXTRACT" else TIME_PARTS
            if not isinstance(word, str) or word.lower() not in known:
                raise ValueError(f"{fn}: unknown {'field' if fn == 'EXTRACT' else 'part'} {word!r}: {e}")
            word = word.lower()
        unit = self._calendar_unit(e, args[0])
        if fn == "DATEDIFF":
            unit_b = self._calendar_unit(e, args[1])
            code = TIME_PARTS.index(word)
            ca, na = self.compile(args[0])
            self.emit(K.X_TS_INDEX, imm=code | unit << 8)
            tmp = self.alloc()
            self.emit(K.X_ST, K.XK_NONE, tmp)
            cb, nb = self.compile(args[1])
            self.emit(K.X_TS_INDEX, imm=code | unit_b << 8)
            self.emit(K.X_SUB_I, K.XK_REG, tmp)
            self.release(tmp)
            return "i", na or nb or "n" in (ca, cb)
        if fn == "ADD_MONTHS":
            cn = self._static_cls(args[1])
            if cn not in ("i", "n"):
                raise ValueError(f"ADD_MONTHS: the number of months must be an integer: {e}")
            leaf = self._leaf(args[1])
            if leaf is not None:
                cls, nullable = self.compile(args[0])
                self._emit_with(K.X_TS_ADDMON, leaf, "i", unit << K.XF_UNIT_SHIFT)
                return "i", nullable or leaf[4]
            _, nn = self.compile(args[1])
            tmp = self.alloc()
            self.emit(K.X_ST, K.XK_NONE, tmp)
            cls, nullable = self.compile(args[0])
            self.emit(K.X_TS_ADDMON, K.XK_REG, tmp, unit << K.XF_UNIT_SHIFT)
            self.release(tmp)
            return "i", nullable or nn
        cls, nullable = self.compile(args[0])
        if cls == "n":
            return "n", True
        if fn == "DATE_TRUNC":
            self.emit(K.X_TS_TRUNC, imm=TIME_PARTS.index(word) | unit << 8)
            return "i", nullable
        if word == "epoch":  # one IEEE operation on the stored value
            self.emit(K.X_I2F)
            if unit == K.TU_DAY:
                self.emit(K.X_MUL_F, K.XK_IMM, 0, 0, _f64_bits(86400.0))
            else:
                self.emit(K.X_DIV_F, K.XK_IMM, 0, 0, _f64_bits(float(_PER_US[K.TU_S][1] * _PER_US[unit][0] // _PER_US[unit][1])))
            return "f", nullable
        self.emit(K.X_TS_PART, imm=TIME_FIELDS.index(word) | unit << 8)
        return "i", nullable

    def _node(self, e: ColumnExpr) -> Tuple[str, bool]:  # noqa: C901
        if is_string_build(e):
            raise NotImplementedError(f"{e} builds a string: it is a whole output column, or the operand of == / != "
                                      f"with a string literal, IS NULL, LIKE or LENGTH")
        if e.kind == Kind.WILDCARD:
            raise ValueError("'*' can't be evaluated as a value")
        if e.kind == Kind.AGG:
            raise ValueError(f"aggregation {e} in a row-wise expression")
        if e.kind in (Kind.NAMED, Kind.LITERAL):
            if e.kind == Kind.LITERAL and isinstance(e.value, str):
                raise NotImplementedError(f"string literal {e} outside a comparison with a string column")
            bare = e.cast(None) if e.as_type is not None else e
            leaf = self._leaf(bare)
            assert leaf is not None
            self._emit_with(K.X_MOV, leaf, leaf[3])
            return leaf[3], leaf[4]
        if e.kind == Kind.UNARY:
            if e.op in ("IS_NULL", "NOT_NULL") and is_string_build(e.col):
                self.string_codes(e.col)
                self.emit(K.X_IS_NULL if e.op == "IS_NULL" else K.X_NOT_NULL)
                return "b", False
            cls, nullable = self.compile(e.col)
            if e.op in ("IS_NULL", "NOT_NULL"):  # string columns are fine here: only validity is read
                self.emit(K.X_IS_NULL if e.op == "IS_NULL" else K.X_NOT_NULL)
                return "b", False
            if cls == "s":
                raise NotImplementedError(f"{e.op} on a string expression: {e}")
            if e.op == "-":
                if cls == "n":
                    return cls, True
                self.emit(K.X_NEG_F if cls == "f" else K.X_NEG_I)
                return ("i" if cls == "b" else cls), nullable
            if e.op == "~":
                self._acc_to(cls, "b")
                self.emit(K.X_NOT)
                return "b", nullable
            raise NotImplementedError(f"unary operator {e.op}")
        if e.kind == Kind.BINARY:
            r = self._temporal_operands(e)
            return self._binary(r) if r.kind == Kind.BINARY else self._node(r)
        if e.kind == Kind.CALL:
            if _scalar(e)[0] is None:
                raise NotImplementedError(f"function {e.func} has no device implementation")
            e = _canonical(e)
            if e.kind != Kind.CALL:
                return self._node(e)
            e = self._temporal_operands(e)
            fn, s = _scalar(e)
            if s.family == "temporal":
                return self._temporal_function(e, fn)
            if s.family in ("string", "regex"):  # the string-building ones were refused above
                return self._string_function(e, fn)
            if fn == "POWER":
                return self._binary(ColumnExpr(Kind.BINARY, "**", e.args))
            if s.family == "numeric":
                return self._unary_function(e, fn)
            if fn == "COALESCE":
                return self._coalesce(e)
            return self._case(e) if fn == "CASE" else self._greatest(e, fn)
        raise NotImplementedError(f"can't evaluate {e!r}")

    def _binary(self, e: ColumnExpr) -> Tuple[str, bool]:
        op = e.op
        if op not in self._REVERSE:
            raise NotImplementedError(f"operator {op}")
        str_cmp = self._string_compare(e)
        if str_cmp is not None:
            return str_cmp
        cl, cr = self._static_cls(e.left), self._static_cls(e.right)
        if "s" in (cl, cr):
            raise NotImplementedError(f"operator {op} on string operands: {e}")
        logical = op in ("&", "|")
        ctx = "b" if logical else ("f" if (op in ("/", "**") or "f" in (cl, cr)) else "i")
        res = "b" if (logical or op in ("<", "<=", ">", ">=", "==", "!=")) else ctx

        def usable(leaf: Any) -> bool:  # a leaf whose class needs no instruction of its own in this context
            return leaf is not None and (not logical or leaf[3] in ("b", "n"))

        def code(o: str) -> int:
            if logical:
                return K.X_AND if o == "&" else K.X_OR
            oi, of = self._OPS[o]
            return of if ctx == "f" else oi

        makes_null = op in ("%", "**")  # x % 0 and a domain error of POWER are NULL whatever the operands
        lr, ll = self._leaf(e.right), self._leaf(e.left)
        if usable(lr):
            ca, na = self.compile(e.left)
            self._acc_to(ca, ctx)
            self._emit_with(code(op), lr, ctx)
            return res, na or lr[4] or makes_null
        if usable(ll):
            cb, nb = self.compile(e.right)
            self._acc_to(cb, ctx)
            self._emit_with(code(self._REVERSE[op]), ll, ctx)
            return res, nb or ll[4] or makes_null
        ca, na = self.compile(e.left)
        self._acc_to(ca, ctx)
        tmp = self.alloc()
        self.emit(K.X_ST, K.XK_NONE, tmp)
        cb, nb = self.compile(e.right)
        self._acc_to(cb, ctx)
        self.emit(code(self._REVERSE[op]), K.XK_REG, tmp)
        self.release(tmp)
        return res, na or nb or makes_null

    def _string_compare(self, e: ColumnExpr) -> Optional[Tuple[str, bool]]:
        """``strcol == 'lit'`` / ``!=``: compare dictionary codes; a string expression's codes are those of its
        new dictionary."""
        t = self.t
        sides = [e.left, e.right]
        named = [s.kind == Kind.NAMED and s.as_type is None and s.name in t.schema
                 and _is_str(t.schema[s.name].type) for s in sides]
        built = [is_string_build(s) and (s.as_type is None or _is_str(s.as_type)) for s in sides]
        lits = [s.kind == Kind.LITERAL and isinstance(s.value, str) and (s.as_type is None or _is_str(s.as_type))
                for s in sides]
        if not (any(named) or any(lits) or any(built)):
            return None
        if e.op not in ("==", "!="):
            raise NotImplementedError(f"operator {e.op} on strings (only == and != run on the device): {e}")
        if (built[0] and lits[1]) or (built[1] and lits[0]):
            s, lit_ = (sides[0], sides[1]) if built[0] else (sides[1], sides[0])
            d, nullable = self.string_codes(s)
            code = d.index(lit_.value).as_py() if len(d) > 0 else -1
            self.emit(K.X_EQ_I if e.op == "==" else K.X_NE_I, K.XK_IMM, 0, 0, code & ((1 << 64) - 1))
            return "b", nullable
        if named[0] and lits[1]:
            c, lit_ = sides[0], sides[1]
        elif named[1] and lits[0]:
            c, lit_ = sides[1], sides[0]
        else:
            raise NotImplementedError(f"string comparison needs a string column and a literal: {e}")
        ci = t.schema.index_of_key(c.name)
        d = t.dictionaries[c.name]
        code = d.index(lit_.value).as_py() if len(d) > 0 else -1  # -1: value not in the dictionary
        self.emit(K.X_MOV, K.XK_COL, self.col_slot(ci))
        self.emit(K.X_EQ_I if e.op == "==" else K.X_NE_I, K.XK_IMM, 0, 0,
                  (code if code is not None else -1) & ((1 << 64) - 1))
        return "b", t.valid[ci] is not None

    def string_codes(self, s: ColumnExpr) -> Tuple[pa.Array, bool]:
        """A string-building expression's int32 codes into the accumulator: the column's code, then the
        result's code in the new dictionary (and, after a CONCAT, the code of a NULL row's result).  Returns
        (the new dictionary, nullable)."""
        t = self.t
        if s.as_type is not None and not _is_str(s.as_type):
            raise NotImplementedError(f"cast of a string expression to {s.as_type}: {s}")
        name, steps = ST.string_chain(s, t.dictionaries)
        r = ST.evaluate(t.dictionaries[name], t.device, steps)
        key: Any = ("STR", name, steps)
        self.tables[key] = (r.remap, r.remap_valid)
        ci = t.schema.index_of_key(name)
        self.emit(K.X_MOV, K.XK_COL, self.col_slot(ci))
        self.emit(K.X_LOOKUP, K.XK_COL, self.col_slot(key), 0, len(t.dictionaries[name]))
        row_null = t.valid[ci] is not None
        if r.null_code is not None and row_null:
            self.emit(K.X_COALESCE, K.XK_IMM, 0, 0, r.null_code)
            row_null = False
        return r.dictionary, row_null or r.remap_valid is not None

    def _string_function(self, e: ColumnExpr, fn: str) -> Tuple[str, bool]:
        """``LIKE`` / ``LENGTH`` of a string column: the code, then its dictionary entry's result.  Of a string
        expression: its code in the new dictionary, then that entry's result."""
        t = self.t
        s = e.args[0] if e.args else None
        if isinstance(s, ColumnExpr) and is_string_build(s):
            return self._string_function_of_expr(e, fn, s)
        if not (isinstance(s, ColumnExpr) and s.kind == Kind.NAMED and s.as_type is None and s.name in t.schema
                and _is_str(t.schema[s.name].type)):
            raise NotImplementedError(f"{fn} needs a string column as its operand: {e}")
        d = t.dictionaries[s.name]
        if fn in REGEX_PREDICATES:
            pattern = _regex_pattern(e, fn)
            if pattern is None:
                return self._node(_lit(None))
            key: Any = ("REGEX", s.name, pattern, fn == "REGEXP_FULL_MATCH")
            if key not in self.tables:
                self.tables[key] = ST.regex_table(d, t.device, pattern, key[3])
        elif fn == "LIKE":
            pattern, escape = _like_pattern(e)
            key = ("LIKE", s.name, pattern, escape)
            if key not in self.tables:
                self.tables[key] = ST.like_table(d, t.device, pattern, escape)
        else:
            key = ("LENGTH", s.name)
            if key not in self.tables:
                self.tables[key] = ST.length_table(d, t.device)
        ci = t.schema.index_of_key(s.name)
        self.emit(K.X_MOV, K.XK_COL, self.col_slot(ci))
        self.emit(K.X_LOOKUP, K.XK_COL, self.col_slot(key), 0, len(d))
        return ("i" if fn == "LENGTH" else "b"), t.valid[ci] is not None or self.tables[key][1] is not None

    def _string_function_of_expr(self, e: ColumnExpr, fn: str, s: ColumnExpr) -> Tuple[str, bool]:
        t = self.t
        if fn in REGEX_PREDICATES:
            pattern = _regex_pattern(e, fn)
            if pattern is None:
                return self._node(_lit(None))
        elif fn == "LIKE":
            pattern, escape = _like_pattern(e)
        d, nullable = self.string_codes(s)
        name, steps = ST.string_chain(s, t.dictionaries)
        if fn in REGEX_PREDICATES:
            key: Any = ("REGEX", ("STR", name, steps), pattern, fn == "REGEXP_FULL_MATCH")
            if key not in self.tables:
                self.tables[key] = ST.regex_table(d, t.device, pattern, key[3])
        elif fn == "LIKE":
            key = ("LIKE", ("STR", name, steps), pattern, escape)
            if key not in self.tables:
                self.tables[key] = ST.like_table(d, t.device, pattern, escape)
        else:
            key = ("LENGTH", ("STR", name, steps))
            if key not in self.tables:
                self.tables[key] = ST.length_table(d, t.device)
        if len(d) == 0:  # every result is NULL: a one-entry table that is never read, for a real device pointer
            self.tables[key] = (torch.zeros(1, dtype=torch.int64, device=t.device),
                                torch.zeros(1, dtype=torch.uint8, device=t.device))
        self.emit(K.X_LOOKUP, K.XK_COL, self.col_slot(key), 0, len(d))
        return ("i" if fn == "LENGTH" else "b"), nullable or self.tables[key][1] is not None

    def _coalesce(self, e: ColumnExpr) -> Tuple[str, bool]:
        args = e.args
        probe = [self._static_cls(a) for a in args]
        if "s" in probe:
            raise NotImplementedError(f"COALESCE on strings: {e}")
        want = "f" if "f" in probe else ("b" if all(p in ("b", "n") for p in probe) and "b" in probe else "i")
        cls, nullable = self.compile(args[0])
        self._acc_to(cls, want)
        for a in args[1:]:
            leaf = self._leaf(a)
            if leaf is not None and (want != "b" or leaf[3] in ("b", "n")):
                self._emit_with(K.X_COALESCE, leaf, want)
                nullable = nullable and leaf[4]
                continue
            tmp = self.alloc()
            self.emit(K.X_ST, K.XK_NONE, tmp)
            cls, n = self.compile(a)
            self._acc_to(cls, want)
            self.emit(K.X_RCOALESCE, K.XK_REG, tmp)  # acc <- tmp if tmp is not NULL else acc
            self.release(tmp)
            nullable = nullable and n
        return want, nullable

    def _case(self, e: ColumnExpr) -> Tuple[str, bool]:
        """CASE WHEN c1 THEN v1 ... ELSE e END: the ELSE first, then the branches from last to first, each
        ``acc <- c TRUE ? v : result so far`` (FB_X_SEL).  A leaf ELSE is read as the operand of the first select."""
        args = list(e.args)
        if len(args) % 2 == 0:
            raise ValueError(f"CASE needs (condition, value) pairs and an ELSE: {e}")
        results = args[1::2] + [args[-1]]
        probe = [self._static_cls(a) for a in results]
        if "s" in probe:
            raise NotImplementedError(f"CASE with string results outside a whole output column, or with string "
                                      f"columns as results: {e}")
        want = _coalesce_cls(probe)
        pending = self._leaf(args[-1])
        if pending is not None and (want != "b" or pending[3] in ("b", "n")):
            nullable = pending[4]
        else:
            pending = None
            cls, nullable = self.compile(args[-1])
            self._acc_to(cls, want)
        r = None
        for i in range(len(args) // 2 - 1, -1, -1):
            if pending is None:
                if r is None:
                    r = self.alloc()
                self.emit(K.X_ST, K.XK_NONE, r)  # the result so far
            cc, _ = self.compile(args[2 * i])
            if cc == "s":
                raise NotImplementedError(f"CASE condition {args[2 * i]} is a string: {e}")
            self._acc_to(cc, "b")
            c = self.alloc()
            self.emit(K.X_ST, K.XK_NONE, c)
            vc, vn = self.compile(args[2 * i + 1])
            self._acc_to(vc, want)
            if pending is not None:
                self._emit_with(K.X_SEL, pending, want, c << K.XF_COND_SHIFT)
                pending = None
            else:
                self.emit(K.X_SEL, K.XK_REG, r, c << K.XF_COND_SHIFT)
            self.release(c)
            nullable = nullable or vn
        if r is not None:
            self.release(r)
        return want, nullable

    def _unary_function(self, e: ColumnExpr, fn: str) -> Tuple[str, bool]:
        """ABS FLOOR CEIL ROUND keep the class (bool counts as int64); SQRT EXP LN LOG10 give float64."""
        d = round_digits(e.args[1]) if len(e.args) == 2 else 0
        cls, nullable = self.compile(e.args[0])
        if cls == "s":
            raise NotImplementedError(f"{fn} of a string: {e}")
        opi, opf = self._UNARY_FN[fn]
        if opi is None and fn not in ("FLOOR", "CEIL"):  # always float64; a domain error is NULL
            if cls != "n":
                self._acc_to(cls, "f")
                self.emit(opf)
            return "f", nullable if fn == "EXP" else True
        if cls == "n":
            return "n", True
        if cls == "f":
            self.emit(opf, imm=d & ((1 << 64) - 1))
            return "f", nullable
        if fn == "ABS":
            self.emit(opi)
        elif fn == "ROUND" and d < 0:
            self.emit(opi, imm=d & ((1 << 64) - 1))
        return "i", nullable

    def _greatest(self, e: ColumnExpr, fn: str) -> Tuple[str, bool]:
        """GREATEST / LEAST: NULL operands are skipped; NULL only if every operand is NULL."""
        args = e.args
        probe = [self._static_cls(a) for a in args]
        if "s" in probe:
            raise NotImplementedError(f"{fn} on strings: {e}")
        want = _coalesce_cls(probe)
        op = {("GREATEST", "f"): K.X_GREATEST_F, ("LEAST", "f"): K.X_LEAST_F}.get(
            (fn, want), K.X_GREATEST_I if fn == "GREATEST" else K.X_LEAST_I)
        cls, nullable = self.compile(args[0])
        self._acc_to(cls, want)
        for a in args[1:]:
            leaf = self._leaf(a)
            if leaf is not None and (want != "b" or leaf[3] in ("b", "n")):
                self._emit_with(op, leaf, want)
                nullable = nullable and leaf[4]
                continue
            tmp = self.alloc()
            self.emit(K.X_ST, K.XK_NONE, tmp)
            cls, n = self.compile(a)
            self._acc_to(cls, want)
            self.emit(op, K.XK_REG, tmp)  # symmetric: no reverse form
            self.release(tmp)
            nullable = nullable and n
        return want, nullable

    def _static_cls(self, e: ColumnExpr) -> str:
        """Class an expression will evaluate to (without emitting code)."""
        if e.as_type is not None:
            return _cls_of(e.as_type)
        if e.kind == Kind.NAMED:
            if e.name not in self.t.schema:
                raise KeyError(f"column {e.name} is not in {self.t.schema}")
            return _cls_of(self.t.schema[e.name].type)
        if e.kind == Kind.LITERAL:
            v = e.value
            return "n" if v is None else "b" if isinstance(v, bool) else \
                "i" if isinstance(v, (int,) + TEMPORAL_LITERALS) else "f" if isinstance(v, float) else "s"
        if e.kind == Kind.UNARY:
            if e.op in ("IS_NULL", "NOT_NULL", "~"):
                return "b"
            c = self._static_cls(e.col)
            return "i" if c == "b" else c
        if is_string_build(e):
            return "s"
        if _scalar(e)[0] is not None:
            e = _canonical(e)
        if e.kind == Kind.BINARY:
            if e.op in ("+", "-", "*", "/", "%", "**"):
                cs = (self._static_cls(e.left), self._static_cls(e.right))
                return "f" if (e.op in ("/", "**") or "f" in cs) else "i"
            return "b"
        s = _scalar(e)[1]
        if s is None:
            return "i"
        if s.result in ("bool", "float64"):
            return s.result[0]
        if s.result == "extract":
            return "f" if str(e.kwargs.get("field", "")).lower() == "epoch" else "i"
        if s.family == "conditional":
            cs = [self._static_cls(a) for a in result_args(e)]
            return "s" if "s" in cs else _coalesce_cls(cs)
        if s.family == "numeric":  # ABS FLOOR CEIL ROUND keep the class
            c = self._static_cls(e.args[0])
            return "i" if c == "b" else c
        return "i"

    def run(self) -> Tuple[List[torch.Tensor], List[Optional[torch.Tensor]]]:
        t = self.t
        cols = [t.columns[i] if isinstance(i, int) else self.tables[i][0] for i in self.cols]
        valid = [t.valid[i] if isinstance(i, int) else self.tables[i][1] for i in self.cols]
        types = [expr_type(t.schema.types[i]) if isinstance(i, int) else K.T_I64 for i in self.cols]
        return K.eval_expr(t.num_rows, t.device, cols, valid, self.ins, [o[0] for o in self.outs],
                           [o[1] for o in self.outs], col_types=types, out_types=[o[2] for o in self.outs])


def _folded(e: ColumnExpr) -> ColumnExpr:
    """``e``, or the literal it folds to when it is an operator between two temporal literals."""
    if e.kind == Kind.BINARY and e.as_type is None and e.op in ("+", "-"):
        a, b = _folded(e.left), _folded(e.right)
        if _is_temporal_literal(a) and _is_temporal_literal(b):
            return _fold(e.op, a.value, b.value, e)
    return e


def _fold(op: str, a: Any, b: Any, e: ColumnExpr) -> ColumnExpr:
    """``a op b`` of two temporal literals, computed on the host."""
    span_a, span_b = isinstance(a, datetime.timedelta), isinstance(b, datetime.timedelta)
    if not span_a and not span_b:  # a date next to a timestamp is its midnight
        a, b = _EPOCH + _literal_us(a) * _US, _EPOCH + _literal_us(b) * _US
    elif span_a != span_b:
        if op not in ("+", "-") or (op == "-" and span_a):
            raise ValueError(f"operator {op} has no meaning between a point in time and an interval: {e}")
        a = a if span_a else _EPOCH + _literal_us(a) * _US
        b = b if span_b else _EPOCH + _literal_us(b) * _US
    if op == "+" and not (span_a or span_b):
        raise ValueError(f"a date or timestamp can't be added to another: {e}")
    import operator

    fn = {"+": operator.add, "-": operator.sub, "<": operator.lt, "<=": operator.le, ">": operator.gt,
          ">=": operator.ge, "==": operator.eq, "!=": operator.ne}[op]
    return _lit(fn(a, b))


def _default_type(cls: str, e: ColumnExpr, schema: Schema) -> pa.DataType:
    tp = e.infer_type(schema)
    if tp is not None:
        return tp
    return {"i": pa.int64(), "f": pa.float64(), "b": pa.bool_()}.get(cls, pa.int64())


def _format_source(e: ColumnExpr, cls: str, schema: Schema) -> pa.DataType:
    """The arrow type whose text ``CAST(x AS STRING)`` writes: ``x``'s inferred type, or the storage type of the
    class K8 computed it in."""
    tp = e.cast(None).infer_type(schema)
    if tp is None or _cls_of(tp) != cls:
        return {"i": pa.int64(), "f": pa.float64(), "b": pa.bool_()}[cls]
    return tp


_STR_CAST = "__str_cast_"


def _string_casts(t: B200Table, exprs: Sequence[ColumnExpr], top: bool) -> Tuple[B200Table, List[ColumnExpr]]:
    """Every ``CAST(x AS STRING)`` of a value ``x`` that is not a whole output column (``top``: the expressions
    themselves are) evaluated into a dictionary column of a wider table, and the trees rewritten to read it: every
    string consumer (==, LIKE, LENGTH, the string-building functions, casts back) then takes it as a string column.
    Equal casts share one column."""
    prog = _Program(t)
    found: Dict[str, Tuple[str, ColumnExpr]] = {}

    def visit(e: Any, is_top: bool) -> Any:
        if not isinstance(e, ColumnExpr):
            return e
        if not is_top and e.as_type is not None and _is_str(e.as_type) and                 e.kind in (Kind.NAMED, Kind.UNARY, Kind.BINARY, Kind.CALL) and                 prog._static_cls(e.cast(None)) not in ("s", "n"):
            bare = e.alias("")
            fp = bare.fingerprint()
            if fp not in found:
                found[fp] = (f"{_STR_CAST}{len(found)}", bare)
            out = _col(found[fp][0])
            return out.alias(e.as_name) if e.as_name != "" else out
        if e.has_args:
            return ColumnExpr(e.kind, e.head, [visit(a, False) for a in e.args],
                              {k: visit(v, False) for k, v in e.kwargs.items()}, e.is_distinct, e.as_name, e.as_type)
        return e

    new = [visit(e, top) for e in exprs]
    if not found:
        return t, list(exprs)
    if any(n.startswith(_STR_CAST) for n in t.schema.names):
        raise NotImplementedError(f"a column name starting with {_STR_CAST} next to a cast to string")
    extra = project(t, [b.alias(name) for name, b in found.values()])
    fields = [pa.field(n, tp) for n, tp in zip(t.schema.names + extra.schema.names, t.schema.types + extra.schema.types)]
    wide = B200Table(Schema(fields), t.columns + extra.columns, t.valid + extra.valid,
                     {**t.dictionaries, **extra.dictionaries}, t.offsets, t.partition_keys)
    return wide, new


def project(t: B200Table, exprs: Sequence[ColumnExpr]) -> B200Table:
    """Evaluate a SELECT list (no aggregations, wildcards already expanded, every column named)."""
    t, exprs = _string_casts(t, exprs, True)
    n, dev = t.num_rows, t.device
    names = [e.output_name for e in exprs]
    out_cols: List[Any] = [None] * len(exprs)
    out_valid: List[Any] = [None] * len(exprs)
    out_types: List[Any] = [None] * len(exprs)
    dicts: Dict[str, pa.Array] = {}
    str_case: Dict[int, pa.Array] = {}  # output -> dictionary of a CASE with string-literal results
    str_built: Dict[int, pa.Array] = {}  # output -> dictionary of a string-building expression
    formatted: Dict[int, pa.DataType] = {}  # output -> the type a cast to string formats (K14)
    pending: List[Tuple[int, ColumnExpr]] = []
    for i, e in enumerate(exprs):
        if e.kind == Kind.NAMED:
            if e.name not in t.schema:
                raise KeyError(f"column {e.name} is not in {t.schema}")
            ci = t.schema.index_of_key(e.name)
            tp = t.schema.types[ci]
            if e.as_type is None or e.as_type == tp:  # pass through, zero copy
                out_cols[i], out_valid[i], out_types[i] = t.columns[ci], t.valid[ci], tp
                if e.name in t.dictionaries:
                    dicts[names[i]] = t.dictionaries[e.name]
                continue
            if _is_str(tp) and _is_str(e.as_type):
                raise NotImplementedError(f"cast of string column {e.name} to {e.as_type}")
        if e.kind == Kind.LITERAL and isinstance(e.value, str) and e.as_type is not None and not _is_str(e.as_type):
            e = string_literal_cast(e)
        if e.kind == Kind.LITERAL and (isinstance(e.value, str) or e.value is None):
            tp = e.as_type or (pa.string() if isinstance(e.value, str) else None)
            if tp is None:
                raise NotImplementedError(f"NULL literal {e} needs a cast to know its type")
            out_types[i] = tp
            out_cols[i] = torch.zeros(n, dtype=_storage_dtype(tp), device=dev)
            if e.value is None:
                out_valid[i] = torch.zeros(n, dtype=torch.uint8, device=dev)
                if _is_str(tp):
                    dicts[names[i]] = pa.array([], type=pa.string())
            else:
                dicts[names[i]] = pa.array([e.value], type=pa.string())
            continue
        strs = case_string_results(e)
        if strs is not None:
            if e.as_type is not None and not _is_str(e.as_type):
                raise NotImplementedError(f"cast of a string CASE to {e.as_type}: {e}")
            str_case[i] = pa.array(strs, type=pa.string())
            e = _coded_case(e, strs)
        pending.append((i, e))
    # ---- computed columns: as many as fit into one launch at a time
    k = 0
    while k < len(pending):
        prog = _Program(t)
        batch: List[Tuple[int, ColumnExpr, str]] = []
        while k < len(pending):
            i, e = pending[k]
            mark = prog.mark()
            try:
                if is_string_build(e) and (e.as_type is None or _is_str(e.as_type)):  # codes into the result's dictionary
                    str_built[i], nullable = prog.string_codes(e)
                    prog.output(torch.int32, nullable, K.T_I32)
                    out_types[i] = pa.string()
                    batch.append((i, e, "i"))
                    k += 1
                    continue
                if i in str_case:  # int32 codes into the literals' dictionary
                    _, nullable = prog.compile(e, top=True)
                    prog.output(torch.int32, nullable, K.T_I32)
                    out_types[i] = pa.string()
                    batch.append((i, e, "i"))
                    k += 1
                    continue
                cls, nullable = prog.compile(e, top=True)
                if cls == "n":  # a bare NULL-valued expression
                    cls = _cls_of(e.as_type) if e.as_type is not None and not _is_str(e.as_type) else "i"
                tp = e.as_type if e.as_type is not None else _default_type(cls, e, t.schema)
                if _is_str(tp) or _cls_of(tp) != cls:
                    store_tp = {"i": pa.int64(), "f": pa.float64(), "b": pa.bool_()}[cls]
                    if not _is_str(tp):
                        tp = store_tp  # an inferred type of another class than the computed value
                    else:
                        formatted[i] = _format_source(e, cls, t.schema)
                        ST.format_kind(formatted[i])  # NotImplementedError before anything runs
                else:
                    store_tp = tp
                prog.output(_storage_dtype(store_tp), nullable, expr_type(store_tp))
            except _OutOfResources as ex:
                if not batch:
                    raise NotImplementedError(f"expression too large for one device program ({ex}): {e}")
                prog.rollback(mark)
                break
            out_types[i] = tp
            batch.append((i, e, cls))
            k += 1
        cols, valids = prog.run()
        for (i, e, cls), c, v in zip(batch, cols, valids):
            if i in str_case:
                dicts[names[i]] = str_case[i]
            elif i in str_built:
                dicts[names[i]] = str_built[i]
            elif i in formatted:
                c, v, dicts[names[i]] = ST.format_values(c, v, formatted[i], dev)
            out_cols[i], out_valid[i] = c, v
    schema = Schema([pa.field(nm, tp) for nm, tp in zip(names, out_types)])
    return B200Table(schema, out_cols, out_valid, dicts)


def _coded_case(e: ColumnExpr, strs: List[str]) -> ColumnExpr:
    """A CASE / IF / IIF / NULLIF with string-literal results as CASE with their codes in ``strs`` as results."""
    args = list(_canonical(e).args)
    code = {s: j for j, s in enumerate(strs)}
    for j in list(range(1, len(args) - 1, 2)) + [len(args) - 1]:
        if args[j].value is not None:
            args[j] = _lit(code[args[j].value])
    return ColumnExpr(Kind.CALL, "CASE", args, as_name=e.as_name)


def predicate_mask(t: B200Table, condition: ColumnExpr) -> torch.Tensor:
    """uint8 mask: 1 where ``condition`` is TRUE (NULL counts as FALSE, like SQL WHERE)."""
    t, (condition,) = _string_casts(t, [condition], False)
    prog = _Program(t)
    try:
        cls, _ = prog.compile(condition.alias("") if condition.as_name else condition)
        if cls == "s":
            raise ValueError(f"{condition} is not a boolean expression")
        if cls == "n":
            return torch.zeros(t.num_rows, dtype=torch.uint8, device=t.device)
        prog._acc_to(cls, "b")
        prog.output(torch.uint8, False)  # FB_X_OUT stores 0 for NULL
    except _OutOfResources as ex:
        raise NotImplementedError(f"condition too large for one device program ({ex}): {condition}")
    cols, _ = prog.run()
    return cols[0]


def filter_table(t: B200Table, condition: ColumnExpr) -> B200Table:
    """``SELECT * FROM t WHERE condition`` (rows keep their order)."""
    if t.num_rows == 0:
        return t
    idx = K.compact_indices(predicate_mask(t, condition))
    if int(idx.shape[0]) == t.num_rows:
        return B200Table(t.schema, t.columns, t.valid, t.dictionaries)
    cols, valid = K.gather_rows(t.columns, t.valid, idx, False)
    return B200Table(t.schema, cols, valid, t.dictionaries)


def rewrite(e: Any, mapper: Any) -> Any:
    """Copy of the tree with ``mapper(node)`` applied top-down (a non-None result replaces the node,
    keeping the node's alias and cast)."""
    if not isinstance(e, ColumnExpr):
        return e
    rep = mapper(e)
    if rep is not None:
        if e.as_type is not None:
            rep = rep.cast(e.as_type)
        return rep.alias(e.as_name) if e.as_name != "" else rep
    if e.has_args:
        args = [rewrite(a, mapper) for a in e.args]
        kwargs = {k: _rewrite_spec(v, mapper) for k, v in e.kwargs.items()}
        return ColumnExpr(e.kind, e.head, args, kwargs, e.is_distinct, e.as_name, e.as_type)
    return e


def _rewrite_spec(v: Any, mapper: Any) -> Any:
    """A keyword argument rewritten: the expressions of a window spec (tuples of nodes and of (node, ascending)
    pairs) as well."""
    if isinstance(v, tuple):
        return tuple(_rewrite_spec(x, mapper) for x in v)
    return rewrite(v, mapper)


def find_aggs(e: Any, out: List[ColumnExpr]) -> None:
    if not isinstance(e, ColumnExpr):
        return
    if e.kind == Kind.AGG:
        out.append(e)
    elif e.has_args:
        for a in _children(e):
            find_aggs(a, out)
