"""CASE, NULLIF, IF / IIF, IFNULL, %, MOD and the numeric functions without a GPU: builders, printer and parser, the
oracle (oracle/scalar.py) pinned to SQLite, and compiled programs run on the numpy machine model (tests/_func_sim.py)
against the oracle, hand-picked and as 600 seeded random trees."""
import math
import sqlite3

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

import _func_sim as fsim
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200.column import ColumnExpr, Kind, SelectColumns, col, function, functions as ff, lit, null, to_sql
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table, expr_type
from oracle import expressions as OX
from oracle import scalar as OS
from test_expr_compiler import _random, _same, _table
from test_expr_random import _boolean, _literal_only

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _parse(text: str) -> ColumnExpr:
    return _parse_select(text, "t", "SELECT " + text + " FROM t").columns[0]


# ---- builders, printer, parser ----------------------------------------------------------------------------------
ROUND_TRIP = [
    ff.case([(col("a") > 0, col("x"))], 0.5),
    ff.case([(col("a") > 0, 1), (col("b") < 2, 2)]),
    ff.case([(col("a") == 1, "one"), (col("a") == 2, "two")], "many"),
    ff.case([(col("p"), ff.case([(col("a") > 0, 1)], 2))], ff.case([(col("b") > 0, 3)], 4)),
    ff.nullif(col("a"), 0), ff.coalesce(col("g"), 1), col("a") % 7, 7 % col("a"), col("x") % 2.5,
    ff.abs(col("x")), ff.floor(col("x")), ff.ceil(col("x")), ff.round(col("x"), 2), ff.round(col("a"), -3),
    ff.round(col("x")), ff.sqrt(col("x")), ff.exp(col("x")), ff.ln(col("x")), ff.log10(col("x")),
    ff.power(col("x"), 2), ff.greatest(col("a"), col("b"), 3), ff.least(col("x"), col("y")),
    ff.sum(ff.case([(col("x") > 0, col("x"))], 0)),
]


@pytest.mark.parametrize("e", ROUND_TRIP, ids=[str(i) for i in range(len(ROUND_TRIP))])
def test_builder_print_parse_round_trip(e):
    text = to_sql(e)
    assert _parse(text).fingerprint() == e.fingerprint(), text
    assert to_sql(_parse(text)) == text


def test_sql_forms():
    same = {
        "IF(a > 0, 1, 2)": ff.case([(col("a") > 0, 1)], 2),
        "IIF(a > 0, 1, 2)": ff.case([(col("a") > 0, 1)], 2),
        "NULLIF(a, 0)": ff.nullif(col("a"), 0),
        "IFNULL(g, 1)": ff.coalesce(col("g"), 1),
        "MOD(a, 7)": col("a") % 7,
        "a % 7 * 2": (col("a") % 7) * 2,
        "CASE a WHEN 1 THEN 'x' WHEN 2 THEN 'y' END": ff.case([(col("a") == 1, "x"), (col("a") == 2, "y")]),
        "CASE WHEN a > 0 THEN 1 END": ff.case([(col("a") > 0, 1)], None),
        "CEILING(x)": ff.ceil(col("x")), "POW(x, 2)": ff.power(col("x"), 2), "ROUND(x)": ff.round(col("x"), 0),
        "ROUND(x, -2)": ff.round(col("x"), -2),
    }
    for text, e in same.items():
        assert _parse(text).fingerprint() == e.fingerprint(), text
    # END is not an implicit alias; a CASE item takes the alias after END
    st = _parse_select("CASE WHEN a > 0 THEN 1 ELSE 0 END pos, b", "FROM t", "q")
    assert [c.output_name for c in st.columns] == ["pos", "b"]
    with pytest.raises(NotImplementedError):
        _parse("WHEN")
    with pytest.raises(NotImplementedError):
        _parse("a + THEN")


def test_builder_and_parser_errors():
    with pytest.raises(ValueError):
        ff.case([], 1)
    with pytest.raises(ValueError):
        _parse("CASE ELSE 1 END")
    with pytest.raises(ValueError):
        ff.greatest(col("a"))
    with pytest.raises(ValueError):
        _parse("LEAST(a)")
    with pytest.raises(ValueError):
        ff.round(col("x"), col("a"))
    with pytest.raises(ValueError):
        ff.round(col("x"), 19)
    with pytest.raises(ValueError):
        _parse("ROUND(x, -19)")
    with pytest.raises(ValueError):
        ff.case([(col("a") > 0, "pos")], 0)
    with pytest.raises(ValueError):
        _parse("IF(a > 0, 'pos', 1)")


def test_infer_type():
    s = Schema("a:long,x:double,s:str")
    assert ff.sqrt(col("a")).infer_type(s) == pa.float64()
    assert function("power", col("a"), 2).infer_type(s) == pa.float64()
    assert ff.case([(col("a") > 0, "p")], "n").infer_type(s) == pa.string()
    assert ff.case([(col("a") > 0, 1)], 0).infer_type(s) is None
    assert function("f", col("a")).infer_type(s) is None and function("MY", col("a")).infer_type(s) is None
    assert (col("a") % 2).infer_type(s) is None


# ---- the oracle pinned to SQLite ----------------------------------------------------------------------------------
def _sqlite():
    con = sqlite3.connect(":memory:")
    try:
        con.execute("SELECT sqrt(4), ln(2)").fetchone()
    except sqlite3.OperationalError:
        pytest.skip("this sqlite3 has no math functions")
    return con


def _ints(rng, n):
    edge = [INT64_MIN, INT64_MIN + 1, -1000, -7, -1, 0, 1, 7, 1000, INT64_MAX]
    return edge + [int(v) for v in rng.integers(-10 ** 6, 10 ** 6, n)] + [int(v) for v in rng.integers(-9, 10, n)]


def test_oracle_integer_mod_abs_floor_ceil_match_sqlite():
    con = _sqlite()
    rng = np.random.default_rng(5)
    xs, ys = _ints(rng, 60), _ints(rng, 60)
    for x in xs:
        for y in ys[:: 7]:
            if (x, y) == (INT64_MIN, -1):  # SQLite evaluates this one as a float
                assert OS.mod(x, y, False) == 0
                continue
            assert OS.mod(x, y, False) == con.execute("SELECT ? % ?", (x, y)).fetchone()[0], (x, y)
        if x != INT64_MIN:  # SQLite raises an integer overflow; the engine wraps like unary minus
            assert OS.abs_(x, False) == con.execute("SELECT abs(?)", (x,)).fetchone()[0]
        assert OS.floor(x, False) == con.execute("SELECT floor(?)", (x,)).fetchone()[0]
        assert OS.ceil(x, False) == con.execute("SELECT ceil(?)", (x,)).fetchone()[0]
    assert OS.abs_(INT64_MIN, False) == INT64_MIN


def test_oracle_case_nullif_match_sqlite():
    con = _sqlite()
    vals = [None, 0, 1, 2]
    for c1 in (None, 0, 1):
        for c2 in (None, 0, 1):
            for e in (None, 5):
                got = OS.case([(c1, 10), (c2, 20)], e)
                assert got == con.execute("SELECT CASE WHEN ? THEN 10 WHEN ? THEN 20 ELSE ? END", (c1, c2, e)).fetchone()[0]
                assert OS.case([(c1, 10)], e) == con.execute("SELECT iif(?, 10, ?)", (c1, e)).fetchone()[0]
    for a in vals:
        for b in vals:
            assert OS.nullif(a, b) == con.execute("SELECT nullif(?, ?)", (a, b)).fetchone()[0]


def test_oracle_domain_errors_match_sqlite():
    con = _sqlite()
    for v in (-1.0, -0.5, -1e300, 0.0, 2.0, 1e-300):
        assert OS.sqrt(v) == con.execute("SELECT sqrt(?)", (v,)).fetchone()[0]
        if v != 0.0:  # LN(0): SQLite gives NULL, IEEE and the engine -inf
            want = con.execute("SELECT ln(?)", (v,)).fetchone()[0]
            got = OS.ref_ln(v)
            assert (got is None and want is None) or got == pytest.approx(want, rel=1e-15)
    assert OS.ref_ln(0.0) == -math.inf


def test_oracle_where_sqlite_differs():
    """Pinned to C / IEEE instead of SQLite:
    - float %: SQLite truncates both sides to integers; here it is fmod (5.5 % 2 = 1.5);
    - ABS(-0.0) is +0.0 (fabs clears the sign bit);
    - ROUND(0.49999999999999994) is 0 (C round; SQLite adds 0.5 first and gives 1.0);
    - LN(0) is -inf (SQLite: NULL);
    - GREATEST skips NULLs (DuckDB / Postgres); SQLite's scalar max() returns NULL if any argument is NULL."""
    assert OS.mod(5.5, 2.0, True) == 1.5 and OS.mod(-5.5, 2.0, True) == -1.5
    assert OS.mod(3.0, math.inf, True) == 3.0 and OS.mod(math.inf, 2.0, True) is None
    assert OS.mod(1.0, -0.0, True) is None and OS.mod(math.nan, 0.0, True) is None
    assert math.copysign(1.0, OS.abs_(-0.0, True)) == 1.0
    assert OS.round_(0.49999999999999994, 0, True) == 0.0 and OS.round_(2.5, 0, True) == 3.0
    assert OS.round_(-2.5, 0, True) == -3.0
    assert OS.ref_ln(0.0) == -math.inf
    assert OS.greatest([None, 3, 1], False) == 3 and OS.greatest([None, None], False) is None
    assert OS.greatest([-0.0, 0.0], True) == 0.0 and math.copysign(1, OS.greatest([-0.0, 0.0], True)) == 1
    assert math.copysign(1, OS.greatest([-0.0, 0.0], True, least=True)) == -1
    assert OS.round_(1234, -2, False) == 1200 and OS.round_(-1250, -2, False) == -1300
    assert OS.round_(INT64_MAX, -1, False) == OS.wrap(INT64_MAX + 3)


# ---- the compiler on the machine model ----------------------------------------------------------------------------
def _run_f(t: B200Table, exprs):
    prog = X._Program(t)
    meta = []
    for e in exprs:
        cls, _ = prog.compile(e, top=True)
        cls = "i" if cls == "n" else cls
        prog.output({"i": torch.int64, "f": torch.float64, "b": torch.uint8}[cls], True)
        meta.append(cls)
    cols = [t.columns[i].numpy() for i in prog.cols]
    valid = [None if t.valid[i] is None else t.valid[i].numpy() for i in prog.cols]
    outs, outv = fsim.run(t.num_rows, cols, valid, prog.ins, [o[2] for o in prog.outs],
                          col_types=[expr_type(t.schema.types[i]) for i in prog.cols])
    res = []
    for cls, o, v in zip(meta, outs, outv):
        dt = {"i": "Int64", "f": "Float64", "b": "boolean"}[cls]
        arr = pd.array(o.astype(bool) if cls == "b" else o, dtype=dt)
        arr[v == 0] = pd.NA
        res.append(pd.Series(arr))
    return res, prog


def _oracle(pdf, exprs):
    df, low, added = OS.lower(pdf, list(exprs))
    return OX.select(df, SelectColumns(*low))


HAND = [
    ff.case([(col("x") > 0, col("x"))], 0), ff.case([(col("p"), col("a")), (col("x") < 0, col("b"))]),
    ff.case([(col("a") > 0, col("x"))], col("a")), ff.case([(col("p"), True)], col("x") > 0),
    function("IF", col("a") > 0, col("g"), col("b")), function("iif", col("p"), 1.5, null()),
    ff.nullif(col("a") % 3, 0), ff.nullif(col("x"), col("y")), ff.coalesce(ff.nullif(col("g"), 2), -1),
    col("a") % 7, col("a") % col("b"), 17 % col("g"), col("x") % 0.75, col("x") % col("y"), (col("a") + 1) % (col("b") - 2),
    function("mod", col("a"), 0), ff.abs(col("a")), ff.abs(col("x")), ff.abs(col("p")), ff.floor(col("x")),
    ff.ceil(col("x") * 3), ff.floor(col("a")), ff.round(col("x") * 100, 2), ff.round(col("x"), 0), ff.round(col("x") * 1e4, -2),
    ff.round(col("a"), -1), ff.round(col("a") * 997, -3), function("ROUND", col("x"), 1), ff.sqrt(col("x")),
    ff.sqrt(ff.abs(col("x"))) + ff.round(col("y"), 2), ff.greatest(col("a"), col("b"), col("g")),
    ff.least(col("x"), col("y"), 0.25), ff.greatest(col("g"), null()), ff.least(col("p"), col("x") > 0),
    ff.greatest(col("x") * 2, col("y") - 1), function("abs", col("x")) == ff.abs(col("x")),
    ff.case([(col("a") % 2 == 0, col("x") % 1.5)], ff.abs(col("y"))),
]


def test_compiled_programs_match_oracle():
    pdf = _random(n=3000, seed=11)
    t = _table(pdf)
    named = [e.alias(f"c{i}") for i, e in enumerate(HAND)]
    want = _oracle(pdf, named)
    for e in named:
        got, _ = _run_f(t, [e])
        _same(got[0], want[e.output_name], str(e))


def _num(rng, depth):
    """Numeric trees mixing the new nodes with + - * and COALESCE.  No function that overflows to inf (an infinity
    minus an infinity is a NaN, which the reference's evaluator reads as NULL and the device keeps as NaN)."""
    if depth == 0 or rng.random() < 0.25:
        r = rng.random()
        if r < 0.7:
            return col(["a", "b", "x", "y", "g"][rng.integers(5)])
        return lit(int(rng.integers(-5, 6))) if r < 0.85 else lit(float(np.round(rng.normal() * 3, 2)))
    sub = lambda: _num(rng, depth - 1)  # noqa: E731
    k = rng.integers(12)
    if k == 0:
        return sub() + sub()
    if k == 1:
        return sub() - sub()
    if k == 2:
        return sub() % sub()
    if k == 3:
        return ff.case([(_boolean(rng, depth - 1), sub()) for _ in range(int(rng.integers(1, 3)))],
                       sub() if rng.random() < 0.7 else None)
    if k == 4:
        return ff.nullif(sub(), sub())
    if k == 5:
        return ff.abs(sub())
    if k == 6:
        return [ff.floor, ff.ceil][rng.integers(2)](sub())
    if k == 7:
        return ff.round(sub(), int(rng.integers(-2, 3)))
    if k == 8:
        return ff.sqrt(ff.abs(sub()))
    if k == 9:
        return [ff.greatest, ff.least][rng.integers(2)](*[sub() for _ in range(int(rng.integers(2, 4)))])
    if k == 10:
        return function("IFNULL", sub(), sub())
    return ff.coalesce(sub(), sub())


@pytest.mark.parametrize("seed", range(6))
def test_random_trees_match_oracle(seed):
    rng = np.random.default_rng(2000 + seed)
    pdf = _random(n=400, seed=seed)
    t = _table(pdf)
    checked = skipped = 0
    while checked < 100:
        e = _num(rng, int(rng.integers(1, 5)))
        if rng.random() < 0.3:
            e = e > _num(rng, 1)
        if _literal_only(e):
            continue
        e = e.alias("r")
        try:
            got, prog = _run_f(t, [e])
        except X._OutOfResources:
            skipped += 1
            continue
        _same(got[0], _oracle(pdf, [e])["r"], str(e))
        checked += 1
    assert skipped < 100


# ---- temporaries ----------------------------------------------------------------------------------------------------
def _nested_case(levels: int) -> ColumnExpr:
    """A CASE nested ``levels`` deep in the THEN of a branch that is not the last: every level holds its result so far
    and its condition in two temporaries while the value of that branch is computed."""
    e: ColumnExpr = ff.case([(col("x") > 0, col("a") + 1)], col("b") + 2)
    for i in range(levels - 1):
        e = ff.case([(col("a") > i, col("b") - i), (col("p"), e)], col("a") * 3)
    return e


def test_case_temporaries_limit():
    pdf = _random(n=200, seed=1)
    t = _table(pdf)
    fits = _nested_case(2)
    prog = X._Program(t)
    prog.compile(fits.alias("r"), top=True)
    used = {b for op, kind, b, _, _ in prog.ins if op == K.X_ST}
    assert len(used) == K.EXPR_NREGS  # all four temporaries
    got, _ = _run_f(t, [fits.alias("r")])
    _same(got[0], _oracle(pdf, [fits.alias("r")])["r"], "nested CASE")
    with pytest.raises(X._OutOfResources):
        X._Program(t).compile(_nested_case(3).alias("r"), top=True)


def test_results_that_can_become_null_get_a_validity_mask():
    """``%`` by zero, a domain error, and CASE / NULLIF make NULLs from operands that are never NULL: the program must
    ask for a validity output, or those rows would read as 0."""
    pdf = pd.DataFrame({"a": np.arange(-5, 5, dtype=np.int64), "x": np.linspace(-2, 2, 10)})
    t = _table(pdf)
    for e in (col("a") % col("a"), 7 % col("a"), col("a") % 0, col("x") % col("x"), ff.power(col("x"), 0.5),
              ff.sqrt(col("x")), ff.ln(col("x")), ff.nullif(col("a"), 1), ff.case([(col("a") > 0, 1)])):
        assert X._Program(t).compile(e, top=True)[1], str(e)
    for e in (col("a") + 1, ff.abs(col("a")), ff.round(col("x"), 2), ff.exp(col("x")), ff.greatest(col("a"), 3),
              ff.case([(col("a") > 0, 1)], 0)):
        assert not X._Program(t).compile(e, top=True)[1], str(e)
