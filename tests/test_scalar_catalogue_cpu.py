"""The scalar function catalogue (column.SCALARS) without a GPU: every head and every other spelling gives the same
program on every route (SQL, ``function(name, ...)`` and the ``functions`` builder), argument counts are checked
alike on each, and ``infer_type`` follows the entry's result rule.  Programs are compiled for a table of CPU tensors;
the per-entry string tables that need the device are replaced by placeholders, which the program only names."""
import pyarrow as pa
import pytest
import torch

from fugue_b200 import expr as X
from fugue_b200 import strings as ST
from fugue_b200.column import SCALAR_ALIASES, SCALARS, ColumnExpr, col, function, functions as ff, is_string_build, lit
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table

SCHEMA = Schema([pa.field("i", pa.int64()), pa.field("f", pa.float64()), pa.field("b", pa.bool_()),
                 pa.field("d", pa.date32()), pa.field("ts", pa.timestamp("us")), pa.field("s", pa.string())])
N = 4
T = B200Table(SCHEMA, [torch.arange(N, dtype=torch.int64), torch.zeros(N, dtype=torch.float64),
                       torch.ones(N, dtype=torch.uint8), torch.zeros(N, dtype=torch.int32),
                       torch.zeros(N, dtype=torch.int64), torch.zeros(N, dtype=torch.int32)],
              [None] * 6, {"s": pa.array(["a", "b"])})
i, f, b, d, ts, s = (col(n) for n in ("i", "f", "b", "d", "ts", "s"))

# head -> (SQL call, function(...) arguments and keywords, the builder's node or None)
CALLS = {
    "CASE": ("CASE WHEN b THEN i ELSE f END", [b, i, f], {}, ff.case([(b, i)], f)),
    "NULLIF": ("NULLIF(i, 2)", [i, 2], {}, ff.nullif(i, 2)),
    "COALESCE": ("COALESCE(i, 2)", [i, 2], {}, ff.coalesce(i, 2)),
    "GREATEST": ("GREATEST(i, f)", [i, f], {}, ff.greatest(i, f)),
    "LEAST": ("LEAST(i, f)", [i, f], {}, ff.least(i, f)),
    "ABS": ("ABS(f)", [f], {}, ff.abs(f)),
    "FLOOR": ("FLOOR(f)", [f], {}, ff.floor(f)),
    "CEIL": ("CEIL(f)", [f], {}, ff.ceil(f)),
    "ROUND": ("ROUND(f, 1)", [f, 1], {}, ff.round(f, 1)),
    "MOD": ("MOD(i, 3)", [i, 3], {}, i % 3),
    "SQRT": ("SQRT(f)", [f], {}, ff.sqrt(f)),
    "EXP": ("EXP(f)", [f], {}, ff.exp(f)),
    "LN": ("LN(f)", [f], {}, ff.ln(f)),
    "LOG10": ("LOG10(f)", [f], {}, ff.log10(f)),
    "POWER": ("POWER(f, 2)", [f, 2], {}, ff.power(f, 2)),
    "LIKE": ("LIKE(s, 'a%')", [s, "a%"], {}, s.like("a%")),
    "LENGTH": ("LENGTH(s)", [s], {}, ff.length(s)),
    "UPPER": ("UPPER(s)", [s], {}, ff.upper(s)),
    "LOWER": ("LOWER(s)", [s], {}, ff.lower(s)),
    "SUBSTR": ("SUBSTR(s, 2, 1)", [s, 2, 1], {}, ff.substr(s, 2, 1)),
    "TRIM": ("TRIM(s, 'x')", [s, "x"], {}, ff.trim(s, "x")),
    "LTRIM": ("LTRIM(s, 'x')", [s, "x"], {}, ff.ltrim(s, "x")),
    "RTRIM": ("RTRIM(s, 'x')", [s, "x"], {}, ff.rtrim(s, "x")),
    "REPLACE": ("REPLACE(s, 'a', 'b')", [s, "a", "b"], {}, ff.replace(s, "a", "b")),
    "CONCAT": ("CONCAT(s, '-')", [s, "-"], {}, ff.concat(s, "-")),
    "REGEXP_MATCHES": ("REGEXP_MATCHES(s, 'a+')", [s, "a+"], {}, ff.regexp_matches(s, "a+")),
    "REGEXP_FULL_MATCH": ("REGEXP_FULL_MATCH(s, 'a+')", [s, "a+"], {}, ff.regexp_full_match(s, "a+")),
    "REGEXP_EXTRACT": ("REGEXP_EXTRACT(s, '(a)', 1)", [s, "(a)", 1], {}, ff.regexp_extract(s, "(a)", 1)),
    "REGEXP_REPLACE": ("REGEXP_REPLACE(s, 'a', 'b', 'g')", [s, "a", "b", "g"], {}, ff.regexp_replace(s, "a", "b", "g")),
    "EXTRACT": ("EXTRACT(year FROM d)", [d], {"field": "year"}, ff.extract("year", d)),
    "DATE_TRUNC": ("DATE_TRUNC('month', ts)", [ts], {"part": "month"}, ff.date_trunc("month", ts)),
    "DATEDIFF": ("DATEDIFF('day', d, ts)", [d, ts], {"part": "day"}, ff.datediff("day", d, ts)),
    "ADD_MONTHS": ("ADD_MONTHS(d, 2)", [d, 2], {}, ff.add_months(d, 2)),
}
# the SQL forms that pass a field or a part: their argument counts are SQL syntax, checked by the parser itself
SQL_SYNTAX = {"CASE", "EXTRACT", "DATE_TRUNC", "DATEDIFF"}


@pytest.fixture(autouse=True)
def _host_tables(monkeypatch):
    """Placeholders for the per-entry tables and string results that are computed on the device."""
    table = (torch.zeros(2, dtype=torch.int64), None)
    monkeypatch.setattr(ST, "like_table", lambda *a: table)
    monkeypatch.setattr(ST, "regex_table", lambda *a: table)
    monkeypatch.setattr(ST, "length_table", lambda *a: table)
    monkeypatch.setattr(ST, "evaluate", lambda *a: ST.StringResult(pa.array(["x"]), table[0], None, None))


def _parse(text: str) -> ColumnExpr:
    return _parse_select(text, "t", "SELECT " + text + " FROM t").columns[0]


def _program(e: ColumnExpr):
    """(instructions, loaded columns and tables, result class) of ``e`` as a whole output column."""
    p = X._Program(T)
    if is_string_build(e):
        p.string_codes(e)
        cls = "s"
    else:
        cls, _ = p.compile(e, top=True)
    return p.ins, p.cols, cls


def test_every_head_has_a_case():
    assert set(CALLS) == set(SCALARS)


@pytest.mark.parametrize("head", sorted(SCALARS))
def test_routes_compile_alike(head):
    sql, args, kwargs, built = CALLS[head]
    want = _program(function(head, *args, **kwargs))
    assert _program(_parse(sql)) == want
    assert _program(built) == want
    assert _program(function(head.lower(), *args, **kwargs)) == want


@pytest.mark.parametrize("alias", sorted(SCALAR_ALIASES))
def test_aliases_compile_as_their_head(alias):
    head, arity = SCALAR_ALIASES[alias]
    sql, args, kwargs, _ = CALLS[head]
    if alias in ("IF", "IIF", "IFNULL"):
        args = args[:arity[0]]
        sql = f"{alias}({', '.join(['b', 'i', 'f'] if head == 'CASE' else ['i', '2'])})"
    else:
        sql = alias + sql[len(head):]
    want = _program(function(head, *args, **kwargs))
    assert _program(function(alias, *args, **kwargs)) == want
    assert _program(_parse(sql)) == want


@pytest.mark.parametrize("name", sorted(SCALARS) + sorted(SCALAR_ALIASES))
def test_argument_counts(name):
    head, arity = SCALAR_ALIASES.get(name, (name, None))
    lo, hi = arity or SCALARS[head].arity
    sql, args, kwargs, _ = CALLS[head]
    args = (args * 2)[:lo]
    counts = [lo - 1] + ([] if hi is None else [hi + 1])
    for k in counts:
        bad = args[:k] if k < lo else args + [lit(1)] * (k - len(args))
        with pytest.raises(ValueError):
            _program(function(name, *bad, **kwargs))
        if head not in SQL_SYNTAX or name != head:
            texts = [_text(a) for a in bad]
            with pytest.raises(ValueError):
                _parse(f"{name}({', '.join(texts)})")


def _text(a) -> str:
    if isinstance(a, ColumnExpr):
        return a.name if a.name else _text(a.value)
    return f"'{a}'" if isinstance(a, str) else str(a)


def test_builders_count_their_arguments():
    for make in (ff.coalesce, ff.greatest, ff.least, ff.concat):
        with pytest.raises(ValueError):
            make(*([i] * (SCALARS[make.__name__.upper()].arity[0] - 1)))


@pytest.mark.parametrize("head", sorted(SCALARS))
def test_infer_type_follows_the_result_rule(head):
    _, args, kwargs, _ = CALLS[head]
    got = function(head, *args, **kwargs).infer_type(SCHEMA)
    rule = SCALARS[head].result
    want = {"extract": pa.int64(), "operand": args[0].infer_type(SCHEMA), "case": None, None: None}.get(rule)
    assert got == (want if rule in ("extract", "operand", "case", None) else pa.type_for_alias(rule))
    assert function(head.lower(), *args, **kwargs).infer_type(SCHEMA) == got


def test_infer_type_special_rules():
    assert function("EXTRACT", ts, field="epoch").infer_type(SCHEMA) == pa.float64()
    assert function("DATE_TRUNC", d, part="day").infer_type(SCHEMA) == pa.date32()
    assert ff.case([(b, "x")], None).infer_type(SCHEMA) == pa.string()
    assert function("IIF", b, "x", "y").infer_type(SCHEMA) == pa.string()
    assert ff.nullif(lit("x"), s).infer_type(SCHEMA) == pa.string()
    assert function("SUBSTRING", s, 1).infer_type(SCHEMA) == pa.string()
    assert function("POW", i, 2).infer_type(SCHEMA) == pa.float64()
    for e in (ff.abs(i), ff.round(f, 1), ff.coalesce(i, 2), ff.greatest(i, f), function("MOD", i, 2)):
        assert e.infer_type(SCHEMA) is None


def test_ifnull_takes_two_arguments_on_every_route():
    with pytest.raises(ValueError):
        _program(function("IFNULL", i, 1, 2))
    with pytest.raises(ValueError):
        _parse("IFNULL(i, 1, 2)")


def test_round_digits_must_be_an_int_on_every_route():
    with pytest.raises(ValueError):
        _program(function("ROUND", f, 1.5))
    with pytest.raises(ValueError):
        _parse("ROUND(f, 1.5)")
    with pytest.raises(ValueError):
        ff.round(f, 1.5)
    with pytest.raises(NotImplementedError):  # not a literal at all
        _program(function("ROUND", f, i))


def test_regexp_like_is_regexp_matches():
    assert _program(function("REGEXP_LIKE", s, "a")) == _program(function("REGEXP_MATCHES", s, "a"))
    assert function("regexp_like", s, "a").infer_type(SCHEMA) == pa.bool_()


def test_literal_arguments():
    with pytest.raises(ValueError):  # a literal of the wrong type
        _program(function("SUBSTR", s, "1"))
    with pytest.raises(NotImplementedError):  # not a literal
        _program(function("SUBSTR", s, i))
    with pytest.raises(ValueError):
        ff.trim(s, 1)
    with pytest.raises(NotImplementedError):
        ff.replace(s, s, "x")
