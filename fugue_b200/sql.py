"""``B200SQLEngine``: recognises the two SQL shapes that reach the GPU kernels.

Reference: ``SQLEngine.select(dfs, statement)`` fugue/execution/execution_engine.py:209-238;
``StructuredRawSQL`` fugue/collections/sql.py:48-151 (pieces ``(is_table_ref, text)``);
FugueSQL forwards plain SELECT text to it (fugue/sql/_visitors.py:743-766,
fugue/workflow/workflow.py:2109-2166) and ``ExecutionEngine.aggregate`` reaches it through
``SQLExpressionGenerator`` (fugue/column/sql.py:275-334).  The native engine hands the text to qpd
(native_execution_engine.py:59-66); here:

    SELECT [DISTINCT] <expr [AS a], ...> FROM t [WHERE <expr>] [GROUP BY <expr, ...>] [HAVING <expr>]
             [QUALIFY <expr>] [ORDER BY c [ASC|DESC], ...] [LIMIT n]
        -> parsed into column expressions (fugue_b200.column) and run by ``engine.select``: row-wise
           parts in the device expression evaluator, SUM/COUNT/MIN/MAX/AVG and VAR_SAMP / VARIANCE / VAR_POP /
           STDDEV_SAMP / STDDEV / STDDEV_POP, SKEWNESS / SKEW / SKEWNESS_POP / KURTOSIS / KURT / KURTOSIS_POP and
           CORR / COVAR_POP / COVAR_SAMP / REGR_* in the hash group-by kernel, window functions by the window
           kernels (K9, K10) after a sort per spec; evaluation order FROM, WHERE, GROUP BY, HAVING, windows,
           QUALIFY, the select list, DISTINCT, ORDER BY, LIMIT.  QUALIFY may name output aliases.

Window functions (DESIGN §7p):

    <call> OVER ( [PARTITION BY <expr>, ...] [ORDER BY <expr> [ASC|DESC] [NULLS LAST], ...] [<frame>] )
    <call>  ::= any aggregate above | ROW_NUMBER() | RANK() | DENSE_RANK() | LAG(x[, n[, default]])
              | LEAD(x[, n[, default]]) | PERCENTILE_CONT / PERCENTILE_DISC(q) WITHIN GROUP (ORDER BY x)
              | NTILE(n) | PERCENT_RANK() | CUME_DIST() | FIRST_VALUE(x) | LAST_VALUE(x) | NTH_VALUE(x, n)
              | EWM_MEAN(x, <decay>[, adjust]) | EWM_VAR(x, <decay>[, adjust]) | EWM_STD(x, <decay>[, adjust])
                (n an integer literal >= 1; NTILE, PERCENT_RANK, CUME_DIST and the EWM functions take no frame; the
                value functions respect NULLs: IGNORE NULLS and FROM LAST raise NotImplementedError)
    <decay> ::= alpha | INTERVAL '..' DAY [TO SECOND]
                (pandas' ewm: alpha a numeric literal in (0, 1]; an INTERVAL is the halflife of a time decay over the
                single ORDER BY expression, EWM_MEAN only; adjust a boolean literal, TRUE by default; ignore_na FALSE,
                min_periods 0 and the sample variance)
    <frame> ::= ROWS | RANGE  BETWEEN <bound> AND <bound>  |  ROWS | RANGE <bound>
    <bound> ::= UNBOUNDED PRECEDING | n PRECEDING | CURRENT ROW | n FOLLOWING | UNBOUNDED FOLLOWING
                (a RANGE offset n may be an INTERVAL '..' DAY / DAY TO SECOND literal)

    With ORDER BY and no frame the frame is RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW (peers
    included), without ORDER BY the whole partition.  NULLs sort last in both directions.  A window over a
    GROUP BY reads group keys and aggregates only (``RANK() OVER (ORDER BY SUM(v) DESC)``).  GROUPS frames,
    EXCLUDE, named windows (WINDOW w AS, OVER w) and NULLS FIRST raise NotImplementedError, and so do
    ROW_NUMBER / RANK / DENSE_RANK / NTILE / PERCENT_RANK / CUME_DIST / LAG / LEAD / FIRST_VALUE / LAST_VALUE /
    NTH_VALUE without OVER; a window in WHERE, GROUP BY, HAVING or in another
    window's arguments raises ValueError.
    SELECT * FROM a [[AS] x] [INNER | LEFT [OUTER] | RIGHT [OUTER] | FULL [OUTER] | [LEFT] SEMI | [LEFT] ANTI] JOIN
             b [[AS] y] USING (k, ...) | ON x.k = y.k [AND ...]              -> hash join kernels
    SELECT * FROM a CROSS JOIN b  |  a NATURAL [<kind above>] JOIN b        -> cross product / common columns

    Each equality names one column of each side (by table or alias; ``k = k`` unqualified); a repeated one counts
    once.  A table ``fa.raw_sql`` named (``_0``, ``_1``) and gave no alias may be named by any qualifier.  A join
    without ON / USING (other than CROSS and NATURAL), CROSS or NATURAL with one, ``a OUTER JOIN b``, ``ON a.k = a.k``
    and qualifiers that name no table raise NotImplementedError.  (In the range and as-of conditions below a
    qualifier that names no table takes the side the condition needs, as DESIGN §7q / §7r describe.)
    SELECT * FROM a ASOF [LEFT [OUTER]] JOIN b
             USING (k, ..., t) | ON a.k = b.k [AND ...] AND a.t >= | > | <= | < b.t  -> as-of join (DESIGN §7q)
    SELECT * FROM a [INNER | LEFT [OUTER]] JOIN b
             ON [a.k = b.k AND ...] a.t BETWEEN b.s AND b.e                  -> range join (DESIGN §7r)
             ON [a.k = b.k AND ...] b.s <= | < a.t AND a.t <= | < b.e        (either operand first, any order)

Expressions: + - * / %, comparisons (= == != <> < <= > >=), AND / OR / NOT, IS [NOT] NULL, [NOT] IN (...),
[NOT] BETWEEN, x [NOT] LIKE 'pattern' [ESCAPE 'c'], CAST(x AS type), CASE [x] WHEN .. THEN .. [ELSE ..] END,
COALESCE, IFNULL, NULLIF, IF / IIF, MOD, ABS, FLOOR, CEIL / CEILING, ROUND, SQRT, EXP, LN, LOG10, POWER / POW,
GREATEST, LEAST, LENGTH, UPPER, LOWER, SUBSTR / SUBSTRING, TRIM, LTRIM, RTRIM, REPLACE, CONCAT, a || b,
DATE '..' / TIMESTAMP '..' / INTERVAL '..' DAY | HOUR | MINUTE | SECOND | DAY TO SECOND literals, x + INTERVAL 'n' MONTH | YEAR,
EXTRACT(field FROM x), DATE_PART, YEAR MONTH DAY HOUR MINUTE SECOND QUARTER DAYOFWEEK DAYOFYEAR WEEK, DATE_TRUNC,
DATEDIFF, ADD_MONTHS, literals, `quoted` and table-qualified names.
Regular expressions: x [NOT] RLIKE 'p', REGEXP_MATCHES / REGEXP_LIKE, REGEXP_FULL_MATCH, REGEXP_EXTRACT,
REGEXP_REPLACE; their string literals are read as written (a backslash is a backslash, '' a quote).
Anything else raises NotImplementedError (there is no host SQL fallback in this package).
"""
import datetime
import itertools
import re
from typing import Any, Dict, List, Tuple

import pyarrow as pa

from .column import (_SPEC_ONLY, BIVARIATES, EWM_HEADS, PERCENTILES, VALUE_HEADS, ColumnExpr, Kind, SelectColumns, _nth,
                     _offset_fn, _value_fn, all_cols, check_arity, col, function, functions, has_window, is_agg, lit,
                     null, scalar_head)
from .dataframe import DataFrame

_AGG = r"(SUM|COUNT|MIN|MAX|AVG|MEAN)\s*\(\s*(\*|[A-Za-z_][\w]*)\s*\)"
_IDENT = r"[A-Za-z_][\w]*"


_TEMP_TABLE_EXPR_PREFIX, _TEMP_TABLE_EXPR_SUFFIX = "<tmpdf:", ">"


class TempTableName:
    """A random table name that prints as ``<tmpdf:_XXXXX>`` - the placeholder ``from_expr`` recognises
    (fugue/collections/sql.py:14-21)."""

    def __init__(self) -> None:
        import uuid

        self.key = "_" + uuid.uuid4().hex[:5].upper()

    def __repr__(self) -> str:
        return _TEMP_TABLE_EXPR_PREFIX + self.key + _TEMP_TABLE_EXPR_SUFFIX


class StructuredRawSQL:
    """SQL text as ``(is_table_ref, text)`` pieces plus the dialect it is written in
    (fugue/collections/sql.py:48-151).  ``construct`` joins the pieces with single spaces, table references
    mapped through ``name_map`` (a function, or a dict - names it does not hold stay as they are).  A change
    of dialect needs sqlglot (``transpile_sql``, :24-45), which this image does not have: asking for one
    raises; the engine's own dialect is None, which never transpiles (:99-103)."""

    def __init__(self, statements: Any, dialect: Any = None):
        self._statements: List[Tuple[bool, str]] = [(bool(a), str(b)) for a, b in statements]
        self._dialect = dialect

    @property
    def dialect(self) -> Any:
        return self._dialect

    def __uuid__(self) -> str:
        import json
        import uuid

        return str(uuid.uuid5(uuid.NAMESPACE_OID, json.dumps([self._statements, self._dialect])))

    @staticmethod
    def from_expr(sql: str, prefix: str = _TEMP_TABLE_EXPR_PREFIX, suffix: str = _TEMP_TABLE_EXPR_SUFFIX,
                  dialect: Any = None) -> "StructuredRawSQL":
        pieces: List[Tuple[bool, str]] = []
        pos = 0
        while pos < len(sql):
            start = sql.find(prefix, pos)
            if start < 0:
                pieces.append((False, sql[pos:]))
                break
            if start > pos:
                pieces.append((False, sql[pos:start]))
            end = sql.find(suffix, start + len(prefix))
            if end < 0:
                raise SyntaxError(f"unterminated table reference in {sql!r}")
            pieces.append((True, sql[start + len(prefix):end]))
            pos = end + len(suffix)
        return StructuredRawSQL(pieces, dialect=dialect)

    def construct(self, name_map: Any = None, dialect: Any = None, log: Any = None) -> str:
        if name_map is None:
            rename = lambda x: x  # noqa: E731
        elif isinstance(name_map, dict):
            rename = lambda x: name_map.get(x, x)  # noqa: E731
        else:
            rename = name_map
        text = " ".join(rename(t) if is_ref else t for is_ref, t in self._statements)
        if self._dialect is not None and dialect is not None and self._dialect != dialect:
            raise NotImplementedError(
                f"SQL transpilation {self._dialect} -> {dialect} needs sqlglot, which is not installed")
        return text


class B200SQLEngine:
    """The SQL facet (``SQLEngine``, fugue/execution/execution_engine.py:183-274)."""

    def __init__(self, execution_engine: Any):
        import uuid

        self._engine = execution_engine
        self._uid = "_" + uuid.uuid4().hex[:5] + "_"

    @property
    def execution_engine(self) -> Any:
        return self._engine

    @property
    def log(self) -> Any:
        return self._engine.log

    @property
    def conf(self) -> Any:
        return self._engine.conf

    def to_df(self, df: Any, schema: Any = None) -> Any:
        return self._engine.to_df(df, schema)

    def encode_name(self, name: str) -> str:
        """A table name no other statement of this process uses (:197-198)."""
        return self._uid + name

    def encode(self, dfs: Dict[str, Any], statement: "StructuredRawSQL") -> Tuple[Dict[str, Any], str]:
        """Tables and statement text with the table references renamed consistently (:200-207)."""
        return ({self.encode_name(k): v for k, v in dfs.items()},
                statement.construct(self.encode_name, dialect=self.dialect))

    def table_exists(self, table: str) -> bool:
        raise NotImplementedError("the b200 SQL engine has no table catalogue")

    def load_table(self, table: str, **kwargs: Any) -> Any:
        raise NotImplementedError("the b200 SQL engine has no table catalogue")

    def save_table(self, df: Any, table: str, mode: str = "overwrite", partition_spec: Any = None,
                   **kwargs: Any) -> None:
        raise NotImplementedError("the b200 SQL engine has no table catalogue")

    @property
    def dialect(self) -> Any:
        return None  # no transpile (fugue/collections/sql.py:99-103)

    @property
    def is_distributed(self) -> bool:
        return self._engine.is_distributed

    def select(self, dfs: Dict[str, Any], statement: Any) -> DataFrame:
        sql = statement.construct() if isinstance(statement, StructuredRawSQL) else str(statement)
        sql = re.sub(r"\s+", " ", sql.strip().rstrip(";"))
        tables = {k: self._engine.to_df(v) for k, v in dfs.items()}
        cut = _top_level_from(sql)
        if re.match(r"(?i)^SELECT ", sql) is None or cut is None:
            raise NotImplementedError(f"unsupported SQL: {sql}")
        items, rest = sql[len("SELECT "):cut[0]].strip(), sql[cut[1]:].strip()
        if re.search(r"(?i)\bJOIN\b", rest):
            return self._join(items, rest, tables, sql)
        return self._single(items, rest, tables, sql)

    def _table(self, name: str, tables: Dict[str, DataFrame], sql: str) -> DataFrame:
        name = name.strip().strip("`")
        if name not in tables:
            raise KeyError(f"table {name} is not among {list(tables)} in: {sql}")
        return tables[name]

    def _single(self, items: str, rest: str, tables: Dict[str, DataFrame], sql: str) -> DataFrame:
        st = _parse_select(items, rest, sql)
        df = self._table(st.table, tables, sql)
        cols = list(st.columns)
        hidden: List[str] = []
        if st.group_by:
            # Fugue infers the GROUP BY keys from the select list (SelectColumns.group_keys); the SQL
            # text must agree with that, extra keys ride along as hidden columns
            probe = SelectColumns(*cols)
            if not probe.has_agg:
                raise NotImplementedError(f"GROUP BY without aggregates: {sql}")
            inferred = {k.fingerprint() for k in probe.group_keys}
            listed = set()
            for g in st.group_by:
                uid = g.alias("").cast(None).fingerprint()
                listed.add(uid)
                if uid not in inferred:
                    name = f"__fb_g{len(hidden)}"
                    hidden.append(name)
                    cols.append(g.alias(name))
            for k in probe.group_keys:
                if k.fingerprint() not in listed:
                    raise ValueError(f"{k} is neither aggregated nor in GROUP BY: {sql}")
        if st.qualify is not None:
            # QUALIFY: a hidden column of the same SELECT (its windows are evaluated with the select list's), then
            # a filter on it, then DISTINCT; an output alias stands for its expression, an input column for itself
            alias = {c.output_name: c.alias("") for c in cols if c.kind != Kind.WILDCARD and c.output_name != ""}
            from .expr import rewrite

            qualify = rewrite(st.qualify, lambda e: alias[e.name] if e.kind == Kind.NAMED and
                              e.name in alias and e.name not in df.schema else None)
            if not has_window(qualify):
                raise ValueError(f"QUALIFY needs a window function: {sql}")
            cols.append(qualify.alias("__fb_q"))
            hidden.append("__fb_q")
        res = self._engine.select(df, SelectColumns(*cols, arg_distinct=st.distinct and st.qualify is None),
                                  where=st.where, having=st.having)
        if st.qualify is not None:
            res = self._engine.filter(res, col("__fb_q"))
        if hidden:
            res = res[[n for n in res.columns if n not in hidden]]
        if st.distinct and st.qualify is not None:
            res = self._engine.distinct(res)
        if st.order_by:
            from collections import OrderedDict

            from .dataframe import B200DataFrame
            from .sort import sort_table

            sorts = OrderedDict((n, asc) for n, asc in st.order_by)
            for n in sorts:
                if n not in res.schema:
                    raise ValueError(f"ORDER BY {n}: not an output column of: {sql}")
            res = B200DataFrame(sort_table(res.native, sorts, "last"))
        if st.limit is not None:
            from .dataframe import B200DataFrame

            res = B200DataFrame(res.native.slice(0, min(st.limit, res.native.num_rows)))
        return res

    def _join(self, items: str, rest: str, tables: Dict[str, DataFrame], sql: str) -> DataFrame:
        if items.strip() != "*":
            raise NotImplementedError(f"only SELECT * is supported for joins: {sql}")
        m = re.match(rf"(?is)^{_TABLE_AS}\s+ASOF\s+(?:(INNER|LEFT|RIGHT|FULL)(?:\s+OUTER)?\s+)?"
                     rf"JOIN\s+{_TABLE_AS}(?:\s+(USING|ON)\s+(.+))?$", rest)
        if m is not None:
            return self._asof_join(m, tables, sql)
        # a join keyword after a table is not its alias: "a LEFT JOIN b" is a left outer join, "a OUTER JOIN b" no join
        m = re.match(rf"(?is)^{_TABLE_AS}\s+(NATURAL\s+)?((?:INNER|CROSS|LEFT\s+SEMI|LEFT\s+ANTI|SEMI|ANTI|"
                     rf"(?:LEFT|RIGHT|FULL)(?:\s+OUTER)?)\s+)?JOIN\s+{_TABLE_AS}(?:\s+(USING|ON)\s+(.+))?$", rest)
        if m is None:
            raise NotImplementedError(f"unsupported join SQL: {sql}")
        t1, t2 = self._table(m.group(1), tables, sql), self._table(m.group(5), tables, sql)
        kind = re.sub(r"\s+", " ", (m.group(4) or "INNER").strip().upper())
        how = {"INNER": "inner", "CROSS": "cross", "LEFT SEMI": "semi", "SEMI": "semi", "LEFT ANTI": "anti",
               "ANTI": "anti", "LEFT OUTER": "left_outer", "LEFT": "left_outer", "RIGHT OUTER": "right_outer",
               "RIGHT": "right_outer", "FULL OUTER": "full_outer", "FULL": "full_outer"}[kind]
        if m.group(3):  # NATURAL: equality on every column the two tables share
            if how == "cross" or m.group(7):
                raise NotImplementedError(f"NATURAL {kind} JOIN takes no ON or USING and is not CROSS: {sql}")
            return self._engine.join(t1, t2, how=how, on=None)
        if how == "cross":
            if m.group(7):
                raise NotImplementedError(f"CROSS JOIN takes no ON or USING (write INNER JOIN): {sql}")
            return self._engine.join(t1, t2, how=how, on=None)
        if not m.group(7):
            raise NotImplementedError(f"{kind} JOIN needs ON or USING (or write NATURAL JOIN / CROSS JOIN): {sql}")
        cond = m.group(8).strip()
        if m.group(7).upper() == "USING":
            on = list(dict.fromkeys(c.strip().strip("`") for c in cond.strip("() ").split(",")))
            return self._engine.join(t1, t2, how=how, on=on)
        sides = _from_sides(m.group(1), m.group(2), m.group(5), m.group(6))
        rng = _range_condition(cond, sides[0], sides[1])
        if rng is not None:
            if how not in ("inner", "left_outer"):
                raise NotImplementedError(f"a range join is INNER or LEFT [OUTER], not {kind}: {sql}")
            on, at, start, end, closed = rng
            return self._engine.range_join(t1, t2, on=on, at=at, start=start, end=end, how=how, closed=closed)
        on = []
        for part in re.split(r"(?i)\s+AND\s+", cond.strip()):
            mm = re.match(rf"^\(?\s*{_QCOL}\s*=\s*{_QCOL}\s*\)?$", part.strip())
            if mm is None or mm.group(2) != mm.group(4):
                raise NotImplementedError(f"only equi-joins on equally named columns: {sql}")
            if not _equality_sides(mm.group(1), mm.group(3), *sides):
                raise NotImplementedError(f"{part.strip()} does not name one column of each table: {sql}")
            if mm.group(2) not in on:
                on.append(mm.group(2))
        return self._engine.join(t1, t2, how=how, on=on)

    def _asof_join(self, m: Any, tables: Dict[str, DataFrame], sql: str) -> DataFrame:
        """``a ASOF [LEFT] JOIN b ON a.k = b.k AND a.t >= b.t`` (DuckDB's form): equalities on equally named
        columns and one inequality on the as-of column, whose operands name both tables.  ``a.t >= b.t`` is a
        backward search, ``>`` a strict one, ``<=`` / ``<`` forward.  ``USING (k, ..., t)``: equality on every
        column but the last, ``>=`` on the last."""
        t1, t2 = self._table(m.group(1), tables, sql), self._table(m.group(4), tables, sql)
        kind = (m.group(3) or "INNER").upper()
        if kind not in ("INNER", "LEFT"):
            raise NotImplementedError(f"ASOF {kind} JOIN: an as-of join is inner or left outer: {sql}")
        how = "left_outer" if kind == "LEFT" else "inner"
        if m.group(6) is None:
            raise NotImplementedError(f"an as-of join needs ON or USING: {sql}")
        cond = m.group(7).strip()
        if m.group(6).upper() == "USING":
            names = [c.strip().strip("`") for c in cond.strip("() ").split(",")]
            return self._engine.asof_join(t1, t2, on=names[:-1], asof=names[-1], how=how, direction="backward",
                                          allow_exact_matches=True)
        left_names, right_names, _ = _from_sides(m.group(1), m.group(2), m.group(4), m.group(5))
        on: List[str] = []
        ineq: List[Tuple[str, str]] = []
        for part in re.split(r"(?i)\s+AND\s+", cond):
            mm = re.match(rf"^\(?\s*(?:({_IDENT})\.)?({_IDENT})\s*(>=|<=|=|>|<)\s*(?:({_IDENT})\.)?({_IDENT})\s*\)?$",
                          part.strip())
            if mm is None or mm.group(2) != mm.group(5):
                raise NotImplementedError(f"an as-of join compares equally named columns: {sql}")
            if mm.group(3) == "=":
                if not _equality_sides(mm.group(1), mm.group(4), left_names, right_names, _ANY_SIDE):
                    raise NotImplementedError(f"{part.strip()} does not name one column of each table: {sql}")
                on.append(mm.group(2))
                continue
            quals = [(q or "").lower() for q in (mm.group(1), mm.group(4))]
            if "" in quals:
                raise NotImplementedError(f"the as-of inequality must qualify both columns: {sql}")
            sides = _operand_sides(quals, left_names, right_names, _ANY_SIDE)
            if None in sides or sides[0] == sides[1]:
                raise NotImplementedError(f"the as-of inequality must name each table once: {sql}")
            op = mm.group(3)
            if sides[0] == "right":  # b.t <= a.t is a.t >= b.t
                op = {">=": "<=", "<=": ">=", ">": "<", "<": ">"}[op]
            ineq.append((mm.group(2), op))
        if len(ineq) != 1:
            raise NotImplementedError(f"an as-of join needs exactly one inequality, got {len(ineq)}: {sql}")
        asof, op = ineq[0]
        return self._engine.asof_join(t1, t2, on=on, asof=asof, how=how,
                                      direction="backward" if op in (">=", ">") else "forward",
                                      allow_exact_matches=op in (">=", "<="))


_JOIN_WORDS = r"(?:AS|INNER|CROSS|LEFT|RIGHT|FULL|OUTER|SEMI|ANTI|NATURAL|ASOF|JOIN|ON|USING)\b"
_TABLE_AS = rf"(`?{_IDENT}`?)(?:\s+AS)?(?:\s+(?!{_JOIN_WORDS})(`?{_IDENT}`?))?"  # table [[AS] alias]
_QCOL = rf"(?:`?({_IDENT})`?\.)?`?({_IDENT})`?"  # [qualifier.]column


_ANY_SIDE = frozenset(("left", "right"))  # a qualifier that names no table may stand for either side


def _from_sides(t1: str, a1: Any, t2: str, a2: Any) -> Tuple[Any, Any, Any]:
    """(left names, right names, anonymous sides) of ``t1 [AS a1] JOIN t2 [AS a2]``: each side is named by its
    table and its alias, lower-cased.  A side is anonymous when its table has a name ``fa.raw_sql`` generated
    (``_0``, ``_1``, ...: the text never spells it) and no alias; a qualifier of an equi-join's equality that names
    no table may stand for it.  (The range and as-of conditions let such a qualifier stand for either side.)"""
    names, anonymous = [], set()
    for side, t, a in (("left", t1, a1), ("right", t2, a2)):
        t = t.strip("`")
        names.append({t.lower()} | ({a.strip("`").lower()} if a else set()))
        if a is None and re.fullmatch(r"_\d+", t):
            anonymous.add(side)
    return names[0], names[1], anonymous


def _operand_sides(quals: List[str], left_names: Any, right_names: Any, anonymous: Any) -> List[Any]:
    """"left" / "right" for the two qualifiers of a comparison's operands, None where a qualifier names no side.
    A qualifier names a table or its alias.  One that names neither may stand for a side in ``anonymous`` (an
    equi-join's: raw_sql's unaliased tables, see ``_from_sides``; ``_ANY_SIDE`` for the range and as-of
    conditions): the side the other operand does not name, and if neither operand names one the operands are in
    FROM order: left table first."""
    sides = ["left" if q in left_names - right_names else "right" if q in right_names - left_names else None
             for q in quals]
    if sides == [None, None] and quals[0] != quals[1] and set(anonymous) == {"left", "right"}:
        sides = ["left", "right"]
    elif None in sides and sides != [None, None]:
        free = "right" if sides[1 - sides.index(None)] == "left" else "left"
        if free in anonymous:
            sides = [s or free for s in sides]
    return sides


def _equality_sides(q1: Any, q2: Any, left_names: Any, right_names: Any, anonymous: Any) -> bool:
    """Whether ``[q1.]k = [q2.]k`` compares the k of one table with the k of the other.  Unqualified, it does;
    qualified, the qualifiers must name the two sides (``a.k = a.k`` and unknown qualifiers do not)."""
    if q1 is None and q2 is None:
        return True
    return sorted(map(str, _operand_sides([(q1 or "").lower(), (q2 or "").lower()], left_names, right_names,
                                          anonymous))) == ["left", "right"]


_COL = rf"(?:({_IDENT})\.)?({_IDENT})"
_RANGE_FLIP = {">=": "<=", "<=": ">=", ">": "<", "<": ">"}


def _range_condition(cond: str, left_names: Any, right_names: Any) -> Any:
    """(on, at, start, end, closed) of an ON condition that is equalities on equally named columns plus exactly
    one range form on qualified columns: ``a.t BETWEEN b.s AND b.e``, or one lower and one upper bound of the same
    left column by right columns (``b.s <= a.t AND a.t < b.e``, either operand first, in any order).  None for
    any other condition, which the equi-join parser then rejects.  Qualifiers that name no table (raw_sql's
    generated names) take the sides that make the condition a range form, the first of them on the left when
    both ways do; an equality whose qualifiers name the same table is no range form."""
    found = list(re.finditer(rf"(?is)(\bNOT\s+)?\b{_COL}\s+BETWEEN\s+{_COL}\s+AND\s+{_COL}\b", cond))
    cmps: List[Tuple[str, str, str, str, str]] = []  # (qualifier, column, op, qualifier, column)
    if found:
        b = found[0]
        if len(found) > 1 or b.group(1) or None in (b.group(2), b.group(4), b.group(6)):
            return None
        cmps += [(b.group(2), b.group(3), ">=", b.group(4), b.group(5)),
                 (b.group(2), b.group(3), "<=", b.group(6), b.group(7))]
        cond = cond[:b.start()] + "\x00" + cond[b.end():]
    on: List[str] = []
    for part in re.split(r"(?i)\s+AND\s+", cond.strip()):
        part = part.strip()
        if re.match(r"^\(?\s*\x00\s*\)?$", part):
            continue
        mm = re.match(rf"^\(?\s*{_COL}\s*(>=|<=|=|>|<)\s*{_COL}\s*\)?$", part)
        if mm is None:
            return None
        if mm.group(3) == "=":
            if mm.group(2) != mm.group(5) or not _equality_sides(mm.group(1), mm.group(4), left_names, right_names,
                                                                  _ANY_SIDE):
                return None
            if mm.group(2) not in on:
                on.append(mm.group(2))
        elif mm.group(1) is None or mm.group(4) is None:
            return None
        else:
            cmps.append(mm.groups())  # type: ignore[arg-type]
    if len(cmps) != 2:
        return None
    known = {q: "left" for q in left_names - right_names}
    known.update({q: "right" for q in right_names - left_names})
    unknown = list(dict.fromkeys(q.lower() for c in cmps for q in (c[0], c[3]) if q.lower() not in known))
    for sides in itertools.product(("left", "right"), repeat=len(unknown)):
        side = dict(known, **dict(zip(unknown, sides)))
        bounds = {}  # "lower" / "upper" -> (left column, right column, inclusive)
        for qa, ca, op, qb, cb in cmps:
            sa, sb = side[qa.lower()], side[qb.lower()]
            if sa == sb:
                break
            if sa == "right":  # b.s <= a.t is a.t >= b.s
                ca, op, cb = cb, _RANGE_FLIP[op], ca
            bounds.setdefault("lower" if op in (">=", ">") else "upper", []).append((ca, cb, op in (">=", "<=")))
        else:
            lower, upper = bounds.get("lower", []), bounds.get("upper", [])
            if len(lower) == 1 and len(upper) == 1 and lower[0][0] == upper[0][0]:
                closed = {(True, True): "both", (True, False): "left", (False, True): "right",
                          (False, False): "neither"}[(lower[0][2], upper[0][2])]
                return on, lower[0][0], lower[0][1], upper[0][1], closed
    return None


def _top_level_from(sql: str) -> Any:
    """(start, end) of the first `` FROM `` outside parentheses and string literals (the one inside
    ``EXTRACT(field FROM x)`` is not the clause), or None."""
    depth, quote, i = 0, "", 0
    while i < len(sql):
        ch = sql[i]
        if quote:
            if ch == "\\" and quote == "'":
                i += 1
            elif ch == quote:
                quote = ""
        elif ch in "'`":
            quote = ch
        elif ch == "(":
            depth += 1
        elif ch == ")":
            depth -= 1
        elif depth == 0 and sql[i:i + 6].upper() == " FROM " and i > 0:
            return i, i + 6
        i += 1
    return None


def _split_commas(text: str) -> List[str]:
    out, depth, cur = [], 0, []
    for ch in text:
        if ch == "(":
            depth += 1
        elif ch == ")":
            depth -= 1
        if ch == "," and depth == 0:
            out.append("".join(cur))
            cur = []
        else:
            cur.append(ch)
    out.append("".join(cur))
    return out


# ---------------------------------------------------------------------------------------------
# SELECT statement parser (single table) -> column expressions
# ---------------------------------------------------------------------------------------------
class _Select:
    def __init__(self) -> None:
        self.distinct = False
        self.columns: List[ColumnExpr] = []
        self.table = ""
        self.where: Any = None
        self.group_by: List[ColumnExpr] = []
        self.having: Any = None
        self.qualify: Any = None
        self.order_by: List[Tuple[str, bool]] = []
        self.limit: Any = None


_TOKEN = re.compile(r"""\s*(?:
    (?P<num>(?:\d+\.\d*|\.\d+|\d+)(?:[eE][+-]?\d+)?)
  | (?P<str>'(?:[^'\\]|\\.|'')*')
  | (?P<bq>`(?:[^`]|``)*`)
  | (?P<id>[A-Za-z_]\w*)
  | (?P<op>\|\||<=|>=|<>|!=|==|=|<|>|\+|-|\*|/|%|\(|\)|,|\.)
)""", re.X)

_AGG_FUNCS = {"SUM": functions.sum, "COUNT": functions.count, "MIN": functions.min, "MAX": functions.max,
              "AVG": functions.avg, "MEAN": functions.avg, "FIRST": functions.first, "LAST": functions.last,
              "VAR_SAMP": functions.var_samp, "VARIANCE": functions.variance, "VAR_POP": functions.var_pop,
              "STDDEV_SAMP": functions.stddev_samp, "STDDEV": functions.stddev, "STDDEV_POP": functions.stddev_pop,
              "SKEWNESS": functions.skewness, "SKEW": functions.skew, "SKEWNESS_POP": functions.skewness_pop,
              "KURTOSIS": functions.kurtosis, "KURT": functions.kurt, "KURTOSIS_POP": functions.kurtosis_pop}
# CORR(a, b), COVAR_POP / COVAR_SAMP(a, b), REGR_*(y, x): two arguments, in SQL's order
_BIVARIATE_FUNCS = {name: getattr(functions, name.lower()) for name in BIVARIATES}
_CLAUSES = ("WHERE", "GROUP", "HAVING", "QUALIFY", "WINDOW", "ORDER", "LIMIT")
_CASE_WORDS = ("WHEN", "THEN", "ELSE", "END")  # never a column name or an implicit alias
_FIELD_FUNCS = {"YEAR": "year", "MONTH": "month", "DAY": "day", "HOUR": "hour", "MINUTE": "minute", "SECOND": "second",
                "QUARTER": "quarter", "DAYOFWEEK": "dow", "DAYOFYEAR": "doy", "WEEK": "week"}
_MONTHS = "INTERVAL_MONTHS"  # a calendar interval literal: only the operand of + / - next to a date or timestamp
# the trees of the column.SCALARS heads that are not the ``functions`` builder of the same name (CASE: IF / IIF)
_SCALAR_FORMS = {"CASE": lambda c, v, e: functions.case([(c, v)], e), "MOD": lambda a, b: a % b,
                 "LIKE": lambda *args: function("LIKE", *args),
                 "ADD_MONTHS": lambda x, n: functions.add_months(x, n.value if n.kind == Kind.LITERAL and
                                                                 n.as_type is None else n)}


# SQL type names inside CAST(... AS type), as schema types; every other name is read by the schema grammar
_SQL_TYPES = {("bigint",): "long", ("integer",): "int", ("int",): "int", ("smallint",): "short", ("tinyint",): "byte",
              ("real",): "float", ("double",): "double", ("double", "precision"): "double", ("varchar",): "str",
              ("text",): "str", ("boolean",): "bool", ("date",): "date", ("timestamp",): "datetime"}


def _cast_type(toks: List[Tuple[str, str]]) -> Any:
    """The type of ``CAST(x AS <toks>)``: a SQL type name, ``timestamp(unit[, time zone])`` or a schema type
    expression (``long``, ``timestamp(ns,UTC)``, ...)."""
    words = tuple(v.lower() for _, v in toks)
    if words in _SQL_TYPES:
        return _SQL_TYPES[words]
    if len(words) >= 4 and words[:2] == ("timestamp", "(") and words[-1] == ")":
        inner = toks[2:-1]
        cut = next((i for i, t in enumerate(inner) if t == ("op", ",")), len(inner))
        unit = "".join(v for _, v in inner[:cut]).lower()
        tz = "".join(_unquote(v) if k == "str" else v for k, v in inner[cut + 1:]) or None
        return pa.timestamp(unit, tz)
    return "".join(v for _, v in toks).lower()


def _tokenize(text: str, sql: str) -> List[Tuple[str, str]]:
    out: List[Tuple[str, str]] = []
    pos = 0
    text = text.rstrip()
    while pos < len(text):
        m = _TOKEN.match(text, pos)
        if m is None or m.end() == pos:
            raise NotImplementedError(f"can't tokenize {text[pos:pos + 20]!r} in: {sql}")
        kind = m.lastgroup
        out.append((kind, m.group(kind)))
        pos = m.end()
    return out


class _Parser:
    """Recursive descent over the token list; precedence OR < AND < NOT < comparison < + - < * / < || < unary."""

    def __init__(self, tokens: List[Tuple[str, str]], sql: str):
        self.t = tokens
        self.i = 0
        self.sql = sql

    def peek(self, k: int = 0) -> Tuple[str, str]:
        return self.t[self.i + k] if self.i + k < len(self.t) else ("end", "")

    def kw(self, *words: str) -> bool:
        """Consume the keyword sequence if it is next."""
        for k, w in enumerate(words):
            kind, val = self.peek(k)
            if kind != "id" or val.upper() != w:
                return False
        self.i += len(words)
        return True

    def at_kw(self, word: str) -> bool:
        kind, val = self.peek()
        return kind == "id" and val.upper() == word

    def op(self, sym: str) -> bool:
        if self.peek() == ("op", sym):
            self.i += 1
            return True
        return False

    def expect(self, sym: str) -> None:
        if not self.op(sym):
            raise NotImplementedError(f"expected {sym!r} near token {self.i} in: {self.sql}")

    def fail(self, what: str) -> Any:
        raise NotImplementedError(f"{what} in: {self.sql}")

    # ---- expressions
    def expr(self) -> ColumnExpr:
        e = self.and_expr()
        while self.kw("OR"):
            e = e | self.and_expr()
        return e

    def and_expr(self) -> ColumnExpr:
        e = self.not_expr()
        while self.kw("AND"):
            e = e & self.not_expr()
        return e

    def not_expr(self) -> ColumnExpr:
        if self.kw("NOT"):
            return ~self.not_expr()
        return self.comparison()

    def comparison(self) -> ColumnExpr:
        e = self.additive()
        while True:
            if self.kw("IS", "NOT", "NULL"):
                e = e.not_null()
            elif self.kw("IS", "NULL"):
                e = e.is_null()
            elif self.at_kw("NOT") and self.peek(1)[1].upper() in ("IN", "BETWEEN"):
                self.i += 1
                e = ~self._in_or_between(e)
            elif self.at_kw("IN") or self.at_kw("BETWEEN"):
                e = self._in_or_between(e)
            elif self.at_kw("RLIKE") and self.peek(1)[0] == "str":
                self.i += 1
                e = e.rlike(self._raw_string())
            elif self.at_kw("NOT") and self.peek(1)[1].upper() == "RLIKE" and self.peek(2)[0] == "str":
                self.i += 2
                e = ~e.rlike(self._raw_string())
            elif self.kw("NOT", "LIKE"):
                e = ~self._like(e)
            elif self.kw("LIKE"):
                e = self._like(e)
            else:
                kind, val = self.peek()
                if kind == "op" and val in ("=", "==", "!=", "<>", "<", "<=", ">", ">="):
                    self.i += 1
                    r = self.additive()
                    e = {"=": e == r, "==": e == r, "!=": e != r, "<>": e != r, "<": e < r, "<=": e <= r,
                         ">": e > r, ">=": e >= r}[val]
                else:
                    return e

    def _string_literal(self, what: str) -> str:
        kind, val = self.peek()
        if kind != "str":
            raise NotImplementedError(f"{what} takes a string literal, got {val!r} in: {self.sql}")
        self.i += 1
        return _unquote(val)

    def _raw_string(self) -> str:
        """A string literal as written, for a regular expression: only '' is resolved (to a quote), so a backslash
        stays a backslash, as in DuckDB and Postgres."""
        val = self.peek()[1]
        self.i += 1
        return val[1:-1].replace("''", "'")

    def _like(self, e: ColumnExpr) -> ColumnExpr:
        pattern = self._string_literal("LIKE")
        escape = self._string_literal("ESCAPE") if self.kw("ESCAPE") else None
        return e.like(pattern, escape)

    def _in_or_between(self, e: ColumnExpr) -> ColumnExpr:
        if self.kw("IN"):
            self.expect("(")
            res: Any = None
            while True:
                c = e == self.additive()
                res = c if res is None else (res | c)
                if not self.op(","):
                    break
            self.expect(")")
            return res
        self.kw("BETWEEN")
        lo = self.additive()
        if not self.kw("AND"):
            self.fail("BETWEEN without AND")
        hi = self.additive()
        return (e >= lo) & (e <= hi)

    def additive(self) -> ColumnExpr:
        e = self.multiplicative()
        while True:
            if self.op("+"):
                e = self._plus(e, self.multiplicative(), 1)
            elif self.op("-"):
                e = self._plus(e, self.multiplicative(), -1)
            else:
                return e

    def _plus(self, a: ColumnExpr, b: ColumnExpr, sign: int) -> ColumnExpr:
        """``a + b`` / ``a - b``; a calendar interval on the right (or, for ``+``, on the left) adds months."""
        for x, iv in ((a, b), (b, a)):
            if iv.kind == Kind.CALL and iv.head == _MONTHS and (iv is b or sign > 0) and \
                    not (x.kind == Kind.CALL and x.head == _MONTHS):
                return functions.add_months(x, sign * iv.args[0].value)
        return a + b if sign > 0 else a - b

    def multiplicative(self) -> ColumnExpr:
        e = self.concat()
        while True:
            if self.op("*"):
                e = e * self.concat()
            elif self.op("/"):
                e = e / self.concat()
            elif self.op("%"):
                e = e % self.concat()
            else:
                return e

    def concat(self) -> ColumnExpr:
        """``a || b``: tighter than ``*`` and left-associative, as in SQLite."""
        e = self.unary()
        while self.op("||"):
            e = functions.concat_strict(e, self.unary())
        return e

    def unary(self) -> ColumnExpr:
        if self.op("-"):
            kind, val = self.peek()
            if kind == "num":  # a negative literal, not a negated expression
                self.i += 1
                return lit(-_number(val))
            return -self.unary()
        if self.op("+"):
            return self.unary()
        return self.primary()

    def primary(self) -> ColumnExpr:
        kind, val = self.peek()
        if kind == "num":
            self.i += 1
            return lit(_number(val))
        if kind == "str":
            self.i += 1
            return lit(_unquote(val))
        if kind == "op" and val == "(":
            self.i += 1
            e = self.expr()
            self.expect(")")
            return e
        if kind == "bq":
            self.i += 1
            return self._maybe_qualified(val[1:-1].replace("``", "`"))
        if kind == "id":
            up = val.upper()
            if up in ("DATE", "TIMESTAMP", "INTERVAL") and self.peek(1)[0] == "str":
                return self._temporal_literal(up)
            if up == "NULL":
                self.i += 1
                return null()
            if up in ("TRUE", "FALSE"):
                self.i += 1
                return lit(up == "TRUE")
            if up == "CASE":
                return self._case()
            if up in _CASE_WORDS:
                self.fail(f"unexpected {up}")
            if up == "CAST" and self.peek(1) == ("op", "("):
                self.i += 2
                e = self.expr()
                if not self.kw("AS"):
                    self.fail("CAST without AS")
                tp: List[Tuple[str, str]] = []
                depth = 0
                while self.peek()[0] != "end" and (depth > 0 or self.peek() != ("op", ")")):
                    depth += {"(": 1, ")": -1}.get(self.peek()[1], 0) if self.peek()[0] == "op" else 0
                    tp.append(self.peek())
                    self.i += 1
                self.expect(")")
                return e.cast(_cast_type(tp))
            if self.peek(1) == ("op", "("):
                return self._call(up)
            self.i += 1
            return self._maybe_qualified(val)
        return self.fail(f"unexpected token {val!r}")

    def _temporal_literal(self, word: str) -> ColumnExpr:
        """``DATE '2024-01-31'``, ``TIMESTAMP '2024-01-31 12:00:00[.ffffff]'``, ``INTERVAL 'n' DAY | HOUR | MINUTE |
        SECOND``, ``INTERVAL 'd hh:mm:ss[.f]' DAY TO SECOND``, ``INTERVAL 'n' MONTH | YEAR``."""
        text = _unquote(self.peek(1)[1])
        self.i += 2
        shown = f"{word} '{text}'"
        try:
            if word == "DATE":
                return lit(datetime.date.fromisoformat(text.strip()))
            if word == "TIMESTAMP":
                v = datetime.datetime.fromisoformat(text.strip())
                return lit(v if isinstance(v, datetime.datetime) else datetime.datetime(v.year, v.month, v.day))
            kind, unit = self.peek()
            unit = unit.upper() if kind == "id" else ""
            self.i += 1
            if unit in ("MONTH", "YEAR"):
                return function(_MONTHS, lit(int(text.strip()) * (12 if unit == "YEAR" else 1)))
            if unit == "DAY" and self.kw("TO", "SECOND"):
                m = re.fullmatch(r"\s*(-?)(\d+) (\d+):(\d+):(\d+)(?:\.(\d{1,6}))?\s*", text)
                if m is None:
                    raise ValueError("expected 'd hh:mm:ss[.ffffff]'")
                d = datetime.timedelta(days=int(m.group(2)), hours=int(m.group(3)), minutes=int(m.group(4)),
                                       seconds=int(m.group(5)), microseconds=int((m.group(6) or "0").ljust(6, "0")))
                return lit(-d if m.group(1) else d)
            if unit in ("DAY", "HOUR", "MINUTE", "SECOND"):
                return lit(datetime.timedelta(**{unit.lower() + "s": int(text.strip())}))
            raise ValueError(f"unknown interval unit {unit!r}")
        except (ValueError, OverflowError) as ex:
            raise ValueError(f"malformed literal {shown}: {ex} in: {self.sql}") from None

    def _case(self) -> ColumnExpr:
        """``CASE WHEN c THEN v ... [ELSE e] END``, or ``CASE x WHEN a THEN v ...``, the searched form with ``x = a``."""
        self.i += 1
        subject = None if any(self.at_kw(w) for w in ("WHEN", "ELSE", "END")) else self.expr()
        branches = []
        while self.kw("WHEN"):
            c = self.expr()
            if not self.kw("THEN"):
                self.fail("CASE WHEN without THEN")
            branches.append((c if subject is None else subject == c, self.expr()))
        else_ = self.expr() if self.kw("ELSE") else None
        if not self.kw("END"):
            self.fail("CASE without END")
        return functions.case(branches, else_)

    def _maybe_qualified(self, name: str) -> ColumnExpr:
        if self.peek() == ("op", ".") and self.peek(1)[0] in ("id", "bq"):  # table.column
            kind, val = self.peek(1)
            self.i += 2
            name = val[1:-1].replace("``", "`") if kind == "bq" else val
        return col(name)

    def _call(self, fn: str) -> ColumnExpr:
        e = self._window_call(fn) if fn in _SPEC_ONLY or fn in VALUE_HEADS else self._plain_call(fn)
        if self.at_kw("OVER"):
            return self._over(e)
        if e.kind == Kind.WINDOW:
            self.fail(f"{fn} without OVER (...)")
        if e.kind == Kind.AGG and any(has_window(a) for a in e.args):
            raise ValueError(f"a window function inside the aggregation {e} in: {self.sql}")
        return e

    def _window_call(self, fn: str) -> ColumnExpr:
        """``ROW_NUMBER() / RANK() / DENSE_RANK()`` or ``LAG / LEAD(x[, n[, default]])``: n an integer literal,
        default a literal."""
        self.i += 2  # name (
        if fn in ("ROW_NUMBER", "RANK", "DENSE_RANK", "PERCENT_RANK", "CUME_DIST"):
            self.expect(")")
            return getattr(functions, fn.lower())()
        args = [self.expr()]
        while self.op(","):
            args.append(self.expr())
        if fn in VALUE_HEADS and (self.at_kw("IGNORE") or self.at_kw("RESPECT")):
            self.fail(f"{fn}(... {self.peek()[1].upper()} NULLS)")
        self.expect(")")
        if fn in ("NTILE", "FIRST_VALUE", "LAST_VALUE", "NTH_VALUE"):
            return self._value_call(fn, args)
        if fn in EWM_HEADS:
            return self._ewm_call(fn, args)
        if len(args) > 3:
            raise ValueError(f"{fn} takes 1 to 3 arguments, got {len(args)} in: {self.sql}")
        for what, x in zip(("n", "default"), args[1:]):
            if x.kind != Kind.LITERAL or x.as_type is not None:
                raise ValueError(f"{fn}: {what} must be a literal, got {x} in: {self.sql}")
        n = args[1].value if len(args) > 1 else 1
        default = args[2].value if len(args) > 2 else None
        return _offset_fn(fn, args[0], n, default, aggregated=True)

    def _ewm_call(self, fn: str, args: List[ColumnExpr]) -> ColumnExpr:
        """``EWM_MEAN / EWM_VAR / EWM_STD(x, alpha [, adjust])``: alpha a numeric literal in (0, 1], or an ``INTERVAL``
        literal, the halflife of a time decay over the single ORDER BY expression; adjust a boolean literal (TRUE).
        pandas' defaults otherwise: ignore_na FALSE, min_periods 0, the sample variance."""
        if len(args) not in (2, 3):
            raise ValueError(f"{fn} takes 2 or 3 arguments, got {len(args)} in: {self.sql}")
        for what, x in zip(("alpha", "adjust"), args[1:]):
            if x.kind != Kind.LITERAL or x.as_type is not None:
                raise ValueError(f"{fn}: {what} must be a literal, got {x} in: {self.sql}")
        decay, adjust = args[1].value, args[2].value if len(args) > 2 else True
        if not isinstance(adjust, bool):
            raise ValueError(f"{fn}: adjust must be TRUE or FALSE, got {args[2]} in: {self.sql}")
        if isinstance(decay, datetime.timedelta):
            return getattr(functions, fn.lower())(args[0], halflife=decay, adjust=adjust, times=True)
        if isinstance(decay, bool) or not isinstance(decay, (int, float)):
            raise ValueError(f"{fn}: alpha must be a number in (0, 1] or an INTERVAL halflife, got {args[1]} in: "
                             f"{self.sql}")
        return getattr(functions, fn.lower())(args[0], alpha=decay, adjust=adjust)

    def _value_call(self, fn: str, args: List[ColumnExpr]) -> ColumnExpr:
        """``NTILE(n)``, ``FIRST_VALUE(x)``, ``LAST_VALUE(x)`` or ``NTH_VALUE(x, n)`` [FROM FIRST] [RESPECT NULLS]: n an
        integer literal >= 1 (any other literal is a ValueError, an expression NotImplementedError).  IGNORE NULLS and
        FROM LAST raise NotImplementedError."""
        want = {"NTILE": 1, "NTH_VALUE": 2}.get(fn, 1)
        if len(args) != want:
            raise ValueError(f"{fn} takes {want} argument{'s' if want > 1 else ''}, got {len(args)} in: {self.sql}")
        if fn == "NTH_VALUE" and self.kw("FROM"):
            if not self.kw("FIRST"):
                self.fail(f"{fn} ... FROM LAST")
        if self.kw("IGNORE", "NULLS"):
            self.fail(f"{fn} ... IGNORE NULLS")
        self.kw("RESPECT", "NULLS")
        if fn in ("NTILE", "NTH_VALUE"):
            x = args[-1]
            if x.kind == Kind.UNARY and x.head == "-" and x.args[0].kind == Kind.LITERAL:
                x = lit(-x.args[0].value) if isinstance(x.args[0].value, (int, float)) else x
            if x.kind != Kind.LITERAL or x.as_type is not None:
                self.fail(f"{fn} with the non-literal n {x}")
            try:
                n = _nth(fn, x.value)
            except ValueError as ex:
                raise ValueError(f"{ex} in: {self.sql}") from None
            if fn == "NTILE":
                return functions.ntile(n)
            return _value_fn(fn, args[0], {"n": n}, aggregated=True)
        return _value_fn(fn, args[0], {}, aggregated=True)

    def _over(self, e: ColumnExpr) -> ColumnExpr:
        """``<call> OVER ([PARTITION BY e, ..] [ORDER BY e [ASC|DESC] [NULLS LAST], ..] [frame])``.  SQL's default
        frame: with ORDER BY, RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW (the current row's peers
        included), without it the whole partition."""
        self.i += 1  # OVER
        if self.peek() != ("op", "("):
            self.fail("named windows (OVER w)")
        self.i += 1
        partition: List[ColumnExpr] = []
        order: List[Tuple[ColumnExpr, bool]] = []
        if self.kw("PARTITION", "BY"):
            partition.append(self.expr())
            while self.op(","):
                partition.append(self.expr())
        if self.kw("ORDER", "BY"):
            while True:
                x = self.expr()
                asc = not self.kw("DESC")
                if asc:
                    self.kw("ASC")
                if self.kw("NULLS", "FIRST"):
                    self.fail("NULLS FIRST (a window orders NULLs last)")
                self.kw("NULLS", "LAST")
                order.append((x, asc))
                if not self.op(","):
                    break
        frame: Dict[str, Any] = {}
        if self.at_kw("GROUPS"):
            self.fail("GROUPS frames")
        if self.at_kw("ROWS") or self.at_kw("RANGE"):
            unit = self.peek()[1].lower()
            self.i += 1
            if self.kw("BETWEEN"):
                start = self._frame_bound(True)
                if not self.kw("AND"):
                    self.fail("BETWEEN without AND in a frame")
                end = self._frame_bound(False)
            else:  # the short form: ROWS <bound> is BETWEEN <bound> AND CURRENT ROW
                start, end = self._frame_bound(True), 0
            frame[unit] = (start, end)
        elif order and e.head not in _SPEC_ONLY and e.head not in PERCENTILES:
            frame["range"] = (None, 0)
        if self.at_kw("EXCLUDE"):
            self.fail("EXCLUDE in a frame")
        self.expect(")")
        return e.over(partition_by=partition, order_by=order, **frame)

    def _frame_bound(self, start: bool) -> Any:
        """UNBOUNDED PRECEDING / FOLLOWING (None), CURRENT ROW (0), ``x PRECEDING`` (-x), ``x FOLLOWING`` (x); x a
        number or an ``INTERVAL '..' DAY [TO SECOND]`` literal."""
        if self.kw("UNBOUNDED"):
            if self.kw("PRECEDING" if start else "FOLLOWING"):
                return None
            raise ValueError(f"a frame {'starts' if start else 'ends'} at UNBOUNDED "
                             f"{'PRECEDING' if start else 'FOLLOWING'} only, in: {self.sql}")
        if self.kw("CURRENT", "ROW"):
            return 0
        kind, val = self.peek()
        if kind == "num":
            self.i += 1
            x: Any = _number(val)
        elif kind == "id" and val.upper() == "INTERVAL" and self.peek(1)[0] == "str":
            x = self._temporal_literal("INTERVAL")
            if x.kind != Kind.LITERAL or not isinstance(x.value, datetime.timedelta):
                self.fail("a frame offset interval in days, hours, minutes or seconds")
            x = x.value
        else:
            return self.fail("a frame bound")
        if self.kw("PRECEDING"):
            return -x
        if self.kw("FOLLOWING"):
            return x
        return self.fail("a frame offset without PRECEDING or FOLLOWING")

    def _plain_call(self, fn: str) -> ColumnExpr:
        self.i += 2  # name (
        if fn in _AGG_FUNCS:
            distinct = self.kw("DISTINCT")
            if self.op("*"):
                arg: ColumnExpr = all_cols()
            else:
                arg = self.expr()
            self.expect(")")
            if distinct:
                if fn != "COUNT":
                    self.fail(f"{fn}(DISTINCT ...)")
                return functions.count_distinct(arg)
            return _AGG_FUNCS[fn](arg)
        if fn in _BIVARIATE_FUNCS:
            if self.kw("DISTINCT"):
                self.fail(f"{fn}(DISTINCT ...)")
            a = self.expr()
            self.expect(",")
            b = self.expr()
            self.expect(")")
            return _BIVARIATE_FUNCS[fn](a, b)
        if fn == "MEDIAN":
            arg = self.expr()
            self.expect(")")
            return functions.median(arg)
        if fn in ("PERCENTILE_CONT", "PERCENTILE_DISC"):
            # PERCENTILE_CONT(q) WITHIN GROUP (ORDER BY x [ASC]): consumed here, so that GROUP is not read as
            # a GROUP BY clause and WITHIN not as an implicit alias
            q = self._quantile_literal(fn)
            self.expect(")")
            if not self.kw("WITHIN", "GROUP"):
                self.fail(f"{fn}(q) needs WITHIN GROUP (ORDER BY ...)")
            self.expect("(")
            if not self.kw("ORDER", "BY"):
                self.fail(f"{fn} WITHIN GROUP needs ORDER BY")
            arg = self.expr()
            if self.kw("DESC"):
                raise NotImplementedError(f"{fn} WITHIN GROUP (ORDER BY ... DESC) in: {self.sql}")
            self.kw("ASC")
            self.expect(")")
            return functions.percentile_cont(arg, q) if fn == "PERCENTILE_CONT" else functions.percentile_disc(arg, q)
        if fn in ("QUANTILE_CONT", "QUANTILE_DISC"):  # DuckDB's spelling: QUANTILE_CONT(x, q)
            arg = self.expr()
            self.expect(",")
            q = self._quantile_literal(fn)
            self.expect(")")
            return functions.percentile_cont(arg, q) if fn == "QUANTILE_CONT" else functions.percentile_disc(arg, q)
        if fn == "EXTRACT":  # EXTRACT(field FROM x)
            kind, field = self.peek()
            if kind not in ("id", "str") or not (self.peek(1)[0] == "id" and self.peek(1)[1].upper() == "FROM"):
                self.fail("EXTRACT needs (field FROM value)")
            self.i += 2
            arg = self.expr()
            self.expect(")")
            return functions.extract(_unquote(field) if kind == "str" else field, arg)
        # a regular expression's string literals (after the string it tests) are read as written
        scalar = scalar_head(fn)
        raw = scalar is not None and scalar[1].family == "regex"
        args: List[Any] = []
        if not self.op(")"):
            while True:
                args.append(self._raw_string() if raw and args and self.peek()[0] == "str" else self.expr())
                if not self.op(","):
                    break
            self.expect(")")
        if fn in _FIELD_FUNCS or fn in ("DATE_PART", "DATE_TRUNC", "DATEDIFF", "DATE_DIFF"):
            return self._temporal_call(fn, args)
        if scalar is None:
            return function(fn, *args)
        head = check_arity(fn, len(args))  # the builder checks the rest
        return (_SCALAR_FORMS.get(head) or getattr(functions, head.lower()))(*args)

    def _temporal_call(self, fn: str, args: List[Any]) -> ColumnExpr:
        """The SQL forms that pass a field or a part as an argument: YEAR(x) ..., DATE_PART('f', x), DATE_TRUNC('p',
        x), DATEDIFF / DATE_DIFF('p', a, b)."""
        want = 1 if fn in _FIELD_FUNCS else 3 if fn in ("DATEDIFF", "DATE_DIFF") else 2
        if len(args) != want:
            raise ValueError(f"{fn} takes {want} argument(s), got {len(args)} in: {self.sql}")
        if fn in _FIELD_FUNCS:
            return functions.extract(_FIELD_FUNCS[fn], args[0])
        word = args[0]
        if word.kind != Kind.LITERAL or not isinstance(word.value, str):
            raise ValueError(f"{fn} takes a string literal as its first argument, got {word} in: {self.sql}")
        if fn == "DATE_PART":
            return functions.extract(word.value, args[1])
        if fn == "DATE_TRUNC":
            return functions.date_trunc(word.value, args[1])
        return functions.datediff(word.value, args[1], args[2])

    def _quantile_literal(self, fn: str) -> Any:
        kind, val = self.peek()
        if kind != "num":
            self.fail(f"{fn} needs a numeric literal q")
        self.i += 1
        return _number(val)

    # ---- select items / lists
    def item(self) -> ColumnExpr:
        if self.peek() == ("op", "*"):
            self.i += 1
            return all_cols()
        e = self.expr()
        if self.kw("AS"):
            kind, val = self.peek()
            if kind not in ("id", "bq"):
                self.fail("AS without a name")
            self.i += 1
            return e.alias(val[1:-1].replace("``", "`") if kind == "bq" else val)
        kind, val = self.peek()
        if kind == "bq" or (kind == "id" and val.upper() not in _CLAUSES + _CASE_WORDS + ("FROM",)):
            self.i += 1  # implicit alias
            return e.alias(val[1:-1].replace("``", "`") if kind == "bq" else val)
        return e


def _unquote(token: str) -> str:
    """The value of a string literal token: quotes removed, '' and backslash escapes resolved."""
    body = token[1:-1].replace("''", "'")
    return re.sub(r"\\(.)", r"\1", body)


def _number(text: str) -> Any:
    return int(text) if re.fullmatch(r"\d+", text) else float(text)


def _default_alias(e: ColumnExpr) -> ColumnExpr:
    """Name an unnamed select item the way the SQL engines do for the common cases."""
    if e.kind == Kind.WILDCARD or e.output_name != "":
        return e
    if e.kind == Kind.AGG and e.arg.kind == Kind.WILDCARD:
        return e.alias(e.func.lower())          # COUNT(*) -> "count"
    named = e.infer_alias()
    return named


def _parse_select(items: str, rest: str, sql: str) -> _Select:
    st = _Select()
    p = _Parser(_tokenize(items, sql), sql)
    st.distinct = p.kw("DISTINCT")
    while True:
        st.columns.append(_default_alias(p.item()))
        if not p.op(","):
            break
    if p.peek()[0] != "end":
        p.fail(f"unexpected token {p.peek()[1]!r} in the select list")
    p = _Parser(_tokenize(rest, sql), sql)
    kind, val = p.peek()
    if kind == "op" and val == "(":
        p.fail("sub-queries are not on the GPU path")
    if kind not in ("id", "bq"):
        p.fail("FROM needs a table name")
    p.i += 1
    st.table = val.strip("`")
    kind, val = p.peek()  # optional alias
    if p.kw("AS"):
        p.i += 1
    elif kind == "id" and val.upper() not in _CLAUSES:
        p.i += 1
    if p.kw("WHERE"):
        st.where = p.expr()
    if p.kw("GROUP", "BY"):
        while True:
            st.group_by.append(p.expr())
            if not p.op(","):
                break
    if p.kw("HAVING"):
        st.having = p.expr()
    if p.kw("QUALIFY"):
        st.qualify = p.expr()
    if p.at_kw("WINDOW"):
        p.fail("named windows (WINDOW w AS ...)")
    if p.kw("ORDER", "BY"):
        while True:
            kind, val = p.peek()
            if kind not in ("id", "bq"):
                p.fail("ORDER BY takes output column names")
            p.i += 1
            asc = True
            if p.kw("DESC"):
                asc = False
            else:
                p.kw("ASC")
            st.order_by.append((val.strip("`"), asc))
            if not p.op(","):
                break
    if p.kw("LIMIT"):
        kind, val = p.peek()
        if kind != "num" or not val.isdigit():
            p.fail("LIMIT takes an integer")
        p.i += 1
        st.limit = int(val)
    if p.peek()[0] != "end":
        p.fail(f"unsupported SQL near {p.peek()[1]!r}")
    if st.where is not None and is_agg(st.where):
        raise ValueError(f"aggregation in WHERE: {sql}")
    for clause, es in (("WHERE", [st.where]), ("GROUP BY", st.group_by), ("HAVING", [st.having])):
        if any(has_window(e) for e in es):
            raise ValueError(f"a window function in {clause}: windows run after {clause}; filter on them with "
                             f"QUALIFY in: {sql}")
    return st
