"""UPPER, LOWER, SUBSTR, TRIM, REPLACE, CONCAT and || without a GPU: the builders, typing, SQL text and parser,
argument validation, the Python oracle (oracle/string_build.py) against sqlite3, the committed case map against a
regeneration from pyarrow, the K8 programs the compiler emits (run by the numpy machine model with FB_X_LOOKUP,
tests/_lookup_sim.py, over per-entry tables computed by the oracle) against oracle/expressions.py, the rejections,
and the multi-GPU rejection of MIN / MAX of a string expression."""
import importlib.util
import os
import random
import sqlite3
import types

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

import _lookup_sim as lsim
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.column import ColumnExpr, Kind, col, function, lit, null, to_sql, functions as ff
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table, expr_type
from oracle import expressions as ox
from oracle import string_build as osb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# 1-, 2-, 3- and 4-byte code points, case pairs with length changes, spaces and tabs
ALPHABET = ["a", "b", "A", "B", " ", "\t", "é", "É", "ß", "ẞ", "İ", "ı", "€", "中", "😀", "𝄞", "Ω", "ω", "K"]


def _parse_item(text: str) -> ColumnExpr:
    return _parse_select(text, "t", "SELECT " + text + " FROM t").columns[0]


def _parse_where(text: str) -> ColumnExpr:
    return _parse_select("*", "t WHERE " + text, "SELECT * FROM t WHERE " + text).where


# ---- builders, typing, SQL text ------------------------------------------------------------------------
def test_builders_and_types():
    sch = Schema("s:str,v:long")
    for e in [ff.upper("s"), ff.lower(col("s")), ff.substr("s", 2), ff.substr("s", -3, 2), ff.trim("s"),
              ff.ltrim("s", "xy"), ff.rtrim("s"), ff.replace("s", "a", "b"), ff.concat("s", "-"),
              ff.concat_strict(col("s"), "-", col("s")), function("upper", col("s")),
              ColumnExpr(Kind.CALL, "substring", [col("s"), lit(1)])]:
        assert e.infer_type(sch) == pa.string(), str(e)
    e = ff.concat_strict("a", col("s"), "b")
    assert e.kind == Kind.BINARY and e.op == "||" and e.left.op == "||" and e.right.value == "b"
    assert ff.substr("s", 1, None).fingerprint() == ff.substr("s", 1).fingerprint()
    assert ff.substr("s", null()).args[1].value is None


@pytest.mark.parametrize("expr,text", [
    (ff.upper(col("s")), "UPPER(s)"),
    (ff.lower(ff.trim(ff.substr(col("s"), 2))), "LOWER(TRIM(SUBSTR(s,2)))"),
    (ff.substr(col("s"), -3, -2), "SUBSTR(s,-3,-2)"),
    (ff.trim(col("s"), "x'y"), "TRIM(s,'x\\'y')"),
    (ff.ltrim(col("s")), "LTRIM(s)"),
    (ff.rtrim(col("s"), "é"), "RTRIM(s,'é')"),
    (ff.replace(col("s"), "aa", ""), "REPLACE(s,'aa','')"),
    (ff.concat(col("s"), "-", None), "CONCAT(s,'-',NULL)"),
    (ff.concat_strict(ff.upper(col("s")), "-", ff.upper(col("s"))), "(UPPER(s) || '-') || UPPER(s)"),
    (ff.substr(col("s"), null(), 2), "SUBSTR(s,NULL,2)"),
    ((ff.upper(col("s")) == "AB") & ff.lower(col("s")).is_null(), "(UPPER(s)='AB') AND LOWER(s) IS NULL"),
    (ff.length(ff.upper(col("s"))), "LENGTH(UPPER(s))"),
    (ff.upper(col("s")).like("A%"), "UPPER(s) LIKE 'A%'"),
])
def test_printer_parser_round_trip(expr, text):
    assert to_sql(expr) == text
    assert _parse_where(text).fingerprint() == expr.fingerprint()
    assert _parse_where(to_sql(_parse_where(text))).fingerprint() == expr.fingerprint()


def test_parser_forms():
    assert _parse_item("substring(s, 1, 3)").fingerprint() == ff.substr(col("s"), 1, 3).fingerprint()
    assert _parse_item("Upper(s)").fingerprint() == ff.upper(col("s")).fingerprint()
    # || binds tighter than * and + and is left-associative
    got = _parse_where("a || 'x' || b = 'q'")
    assert got.fingerprint() == (ff.concat_strict(col("a"), "x", col("b")) == "q").fingerprint()
    got = _parse_where("v * s || 'x' > 1")
    assert got.fingerprint() == ((col("v") * ff.concat_strict(col("s"), "x")) > 1).fingerprint()
    got = _parse_where("v + s || t = 1")
    assert got.fingerprint() == ((col("v") + ff.concat_strict(col("s"), col("t"))) == 1).fingerprint()
    st = _parse_select("LOWER(s) AS l, COUNT(*) AS n", "t GROUP BY LOWER(s)", "")
    assert st.columns[0].fingerprint() == ff.lower(col("s")).alias("l").fingerprint()
    assert st.group_by[0].fingerprint() == ff.lower(col("s")).fingerprint()


def test_argument_validation():
    for bad in [lambda: ff.substr("s", 1.5), lambda: ff.substr("s", True), lambda: ff.substr("s", 1, "2"),
                lambda: ff.trim("s", 3), lambda: ff.replace("s", 1, "x"), lambda: ff.concat(),
                lambda: ff.concat_strict("s"), lambda: _parse_item("UPPER(s, 1)"), lambda: _parse_item("SUBSTR(s)"),
                lambda: _parse_item("SUBSTR(s, 1, 2, 3)"), lambda: _parse_item("TRIM(s, 'a', 'b')"),
                lambda: _parse_item("REPLACE(s, 'a')"), lambda: _parse_item("LOWER()")]:
        with pytest.raises(ValueError):
            bad()
    for bad in [lambda: ff.substr("s", col("v")), lambda: ff.trim("s", col("c")), lambda: _parse_item("SUBSTR(s, v)")]:
        with pytest.raises(NotImplementedError):
            bad()
    with pytest.raises(ValueError):  # the compiler checks trees that were not made by the builders
        ST.string_chain(ColumnExpr(Kind.CALL, "UPPER", [col("s"), lit(1)]), {"s"})
    with pytest.raises(ValueError):
        ST.string_chain(ColumnExpr(Kind.CALL, "SUBSTR", [col("s"), lit(1.0)]), {"s"})


# ---- the oracle, pinned against sqlite3 ------------------------------------------------------------------
def _random_strings(rng: random.Random, n: int):
    out = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 8))) for _ in range(n)]
    return out + ["", " ", "\t", "  a  ", " \ta\t ", "aaa", "aaaa", None]


def test_oracle_against_sqlite():
    rng = random.Random(11)
    values = _random_strings(rng, 300)
    db = sqlite3.connect(":memory:")

    def q(sql, *args):
        return db.execute("SELECT " + sql, args).fetchone()[0]

    for v in values:
        for a in range(-9, 10):
            assert osb.substr(v, a) == q("substr(?, ?)", v, a), (v, a)
            for b in range(-9, 10):
                assert osb.substr(v, a, b) == q("substr(?, ?, ?)", v, a, b), (v, a, b)
        assert osb.substr(v, None, 2) == q("substr(?, NULL, 2)", v)
        assert osb.substr(v, 1, None) == q("substr(?, 1, NULL)", v)
        for chars in [" ", "a", "aé", "\t ", "", "😀中", None]:
            assert osb.trim(v, chars) == q("trim(?, ?)", v, chars), (v, chars)
            assert osb.ltrim(v, chars) == q("ltrim(?, ?)", v, chars), (v, chars)
            assert osb.rtrim(v, chars) == q("rtrim(?, ?)", v, chars), (v, chars)
        assert osb.trim(v) == q("trim(?)", v) and osb.ltrim(v) == q("ltrim(?)", v) and osb.rtrim(v) == q("rtrim(?)", v)
        for old, new in [("a", "xy"), ("aa", "b"), ("é", ""), ("", "z"), (" ", "_"), ("😀", "中中"), (None, "x"),
                         ("a", None)]:
            assert osb.replace(v, old, new) == q("replace(?, ?, ?)", v, old, new), (v, old, new)
        for parts in [(v, "-"), ("<", v, ">"), (v, None, v), (None,), (v,)]:
            assert osb.concat(*parts) == q("concat(" + ",".join("?" * len(parts)) + ")", *parts), parts
            if len(parts) > 1:
                assert osb.concat_strict(*parts) == q(" || ".join("?" * len(parts)), *parts), parts
    # the examples of the SQLite documentation the semantics are stated with
    assert [osb.substr("hello", 0, 2), osb.substr("hello", -3, 2), osb.substr("hello", 4, -3),
            osb.substr("hello", -10, 3)] == ["h", "ll", "hel", ""]
    assert osb.replace("aaa", "aa", "b") == "ba" and osb.upper("ß") == "ẞ" and osb.lower("İ") == "i"


def test_casemap_matches_pyarrow():
    spec = importlib.util.spec_from_file_location("make_casemap", os.path.join(ROOT, "tools", "make_casemap.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with open(os.path.join(ROOT, "fugue_b200", "csrc", "fb_casemap.inc")) as f:
        assert f.read() == mod.render()
    up, low = mod.mapping(True), mod.mapping(False)
    assert len(up) + 26 == 1506 and len(low) + 26 == 1488
    def width(c):
        return len(chr(c).encode("utf-8"))

    assert sum(width(a) != width(b) for a, b in up) == 34 and sum(width(a) != width(b) for a, b in low) == 27


# ---- the compiler and the machine model ------------------------------------------------------------------
def _apply(step, v):
    name = step[0]
    if name == "NULL":
        return None
    if name == "FORMAT":
        if v is None and not step[2]:
            return None
        out = bytearray()
        for tk in step[1]:
            if tk == K.STR_SELF:
                out += (v or "").encode()
            else:
                out.append(tk)
        return out.decode()
    if v is None:
        return None
    if name == "SUBSTR":
        return osb.substr(v, step[1], "absent" if step[2] is None else step[2])
    if name in ("TRIM", "LTRIM", "RTRIM"):
        return getattr(osb, name.lower())(v, step[1].decode())
    if name == "REPLACE":
        return osb.replace(v, step[1].decode(), step[2].decode())
    return getattr(osb, name.lower())(v)


def _oracle_evaluate(d, device, steps):
    """``strings.evaluate`` restated on the host with the oracle: CPU tensors."""
    vals = d.to_pylist()
    extra = any(s[0] == "FORMAT" and s[2] for s in steps)
    if extra:
        vals = vals + [None]
    for s in steps:
        vals = [_apply(s, v) for v in vals]
    new = list(dict.fromkeys(v for v in vals if v is not None))
    code = {v: i for i, v in enumerate(new)}
    remap = torch.tensor([code.get(v, 0) for v in vals] or [0], dtype=torch.int64)
    remap_valid = None if all(v is not None for v in vals) and vals else \
        torch.tensor([v is not None for v in vals] or [False], dtype=torch.uint8)
    null_code = code[vals[-1]] if extra and vals[-1] is not None else None
    return ST.StringResult(pa.array(new, type=pa.string()), remap, remap_valid, null_code)


def _entry_tables(monkeypatch):
    def valid_of(d):
        return None if d.null_count == 0 else torch.tensor([v is not None for v in d.to_pylist()], dtype=torch.uint8)

    def like_table(d, device, pattern, escape):
        from oracle import strings as ostr
        return torch.tensor([bool(ostr.like(v, pattern, escape)) for v in d.to_pylist()], dtype=torch.int64), valid_of(d)

    def length_table(d, device):
        return torch.tensor([len(v) if v is not None else 0 for v in d.to_pylist()], dtype=torch.int64), valid_of(d)

    monkeypatch.setattr(ST, "evaluate", _oracle_evaluate)
    monkeypatch.setattr(ST, "like_table", like_table)
    monkeypatch.setattr(ST, "length_table", length_table)


def _random_table(rng: np.random.Generator, n: int, ndict: int, null_entries: bool):
    words = set()
    while len(words) < ndict:
        words.add("".join(ALPHABET[int(i)] for i in rng.integers(0, len(ALPHABET), int(rng.integers(0, 7)))))
    entries = sorted(words, key=lambda _: rng.random())
    if null_entries:
        entries[int(rng.integers(0, ndict))] = None
    codes = rng.integers(0, ndict, n).astype(np.int32)
    valid = (rng.random(n) > 0.2).astype(np.uint8)
    v = rng.integers(-5, 5, n).astype(np.int64)
    t = B200Table(Schema("s:str,v:long,t:str"), [torch.from_numpy(codes), torch.from_numpy(v), torch.from_numpy(codes)],
                  [torch.from_numpy(valid), None, None], {"s": pa.array(entries), "t": pa.array(entries)})
    pdf = pd.DataFrame({"s": pd.array([entries[c] if m else None for c, m in zip(codes, valid)], dtype="string"),
                        "v": v})
    return t, pdf


def _run_model(t: B200Table, e: ColumnExpr):
    prog = X._Program(t)
    cls, _ = prog.compile(e, top=True)
    prog.output(torch.uint8 if cls == "b" else torch.int64, True)
    cols = [t.columns[i] if isinstance(i, int) else prog.tables[i][0] for i in prog.cols]
    valid = [t.valid[i] if isinstance(i, int) else prog.tables[i][1] for i in prog.cols]
    types = [expr_type(t.schema.types[i]) if isinstance(i, int) else K.T_I64 for i in prog.cols]
    outs, outv = lsim.run(t.num_rows, [c.numpy() for c in cols], [None if m is None else m.numpy() for m in valid],
                         prog.ins, [K.T_U8 if cls == "b" else K.T_I64], col_types=types)
    return prog, [None if not ok else (bool(x) if cls == "b" else int(x)) for x, ok in zip(outs[0], outv[0])]


def _expected(pdf: pd.DataFrame, e: ColumnExpr):
    df2, (e2,), _ = osb.lower_exprs(pdf, [e])
    v = ox.evaluate(e2, df2)
    return [None if x is pd.NA else (bool(x) if isinstance(x, (bool, np.bool_)) else int(x)) for x in v]


def test_compiler_emits_mov_lookup(monkeypatch):
    _entry_tables(monkeypatch)
    t, _ = _random_table(np.random.default_rng(0), 100, 20, False)
    nested = ff.upper(ff.trim(ff.substr(col("s"), 2)))
    prog, _ = _run_model(t, nested == "A")
    assert [i[0] for i in prog.ins[:3]] == [K.X_MOV, K.X_LOOKUP, K.X_EQ_I] and prog.ins[1][4] == 20
    prog, _ = _run_model(t, ff.length(nested) + ff.length(col("s")))
    ops = [i[0] for i in prog.ins]
    assert ops[:3] == [K.X_MOV, K.X_LOOKUP, K.X_LOOKUP] and ops.count(K.X_LOOKUP) == 3
    prog, _ = _run_model(t, ff.concat(col("s"), "!").is_null())  # a NULL row: the code of '!'
    assert [i[0] for i in prog.ins[:4]] == [K.X_MOV, K.X_LOOKUP, K.X_COALESCE, K.X_IS_NULL]
    prog = X._Program(t)  # a whole output column: the codes of the new dictionary
    d, _ = prog.string_codes(nested)
    assert [i[0] for i in prog.ins] == [K.X_MOV, K.X_LOOKUP] and d.type == pa.string()


@pytest.mark.parametrize("seed", range(4))
def test_model_matches_oracle(monkeypatch, seed):
    _entry_tables(monkeypatch)
    rng = np.random.default_rng(seed)
    t, pdf = _random_table(rng, 2000, int(rng.integers(1, 50)), null_entries=seed % 2 == 1)
    s = col("s")
    exprs = []
    for b in [ff.upper(s), ff.lower(s), ff.substr(s, 2, 3), ff.substr(s, -2), ff.trim(s), ff.ltrim(s, "a "),
              ff.rtrim(s, "\t"), ff.replace(s, "a", "xy"), ff.concat(s, "-", s), ff.concat_strict(s, "!"),
              ff.upper(ff.trim(ff.substr(s, 2))), ff.concat(ff.lower(s), None), ff.concat_strict(s, None),
              ff.substr(s, null()), ff.concat(ff.substr(s, null()), "x"), ff.lower(ff.concat("<", s))]:
        exprs += [b == "A", b != "a", b.is_null(), b.not_null(), ff.length(b), b.like("%a%"),
                  (ff.length(b) > 2) & (col("v") > 0)]
    for e in exprs:
        _, got = _run_model(t, e)
        assert got == _expected(pdf, e), str(e)


def test_compiler_rejections(monkeypatch):
    _entry_tables(monkeypatch)
    t, _ = _random_table(np.random.default_rng(1), 10, 5, False)
    s = col("s")
    for e in [ff.upper(s),                                   # a bare string result is a whole output column
              ff.concat_strict(ff.upper(s), s) == "A",      # different operands
              ff.concat(s, col("t")) == "A",                # two string columns
              ff.concat(s, 1) == "A",                       # a number inside a concatenation
              ff.upper(col("v")) == "A",                    # no string column
              ff.concat("a", "b") == "ab",
              ff.upper(s) < "B", ff.upper(s) >= "B",        # string ordering
              ff.upper(s) == col("t"),
              ff.upper(s.cast(int)) == "A",
              ff.replace(s, "x" * (K.STR_MAX_LITERAL + 1), "") == "",
              ff.case([(col("v") > 0, s)], ff.upper(s)) == "A",
              ColumnExpr(Kind.CALL, "ILIKE", [s, lit("a")]), ColumnExpr(Kind.CALL, "LPAD", [s, lit(3)]),
              ColumnExpr(Kind.CALL, "INSTR", [s, lit("a")]), ColumnExpr(Kind.CALL, "LEFT", [s, lit(1)])]:
        with pytest.raises(NotImplementedError):
            X._Program(t).compile(e, top=True)


def test_project_rejects_string_expression_casts(monkeypatch):
    _entry_tables(monkeypatch)
    t, _ = _random_table(np.random.default_rng(2), 10, 5, False)
    with pytest.raises(NotImplementedError):
        X._Program(t).string_codes(ff.upper(col("s")).cast(int))


# ---- multi-GPU: MIN / MAX of a string expression stays unsupported ------------------------------------------
def test_distributed_string_expression_min_max_raises():
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.dist import DistributedB200Engine
    from fugue_b200.partition import PartitionSpec

    t = B200Table(Schema("k:long,s:str"), [torch.tensor([1, 2]), torch.tensor([0, 1], dtype=torch.int32)], None,
                  {"s": pa.array(["x", "y"])})
    fake = types.SimpleNamespace(_world=2, to_df=lambda df: df)
    for fn in (ff.min, ff.max):
        for arg in (ff.upper(col("s")), ff.concat_strict(col("s"), "!"), ff.substr(col("s"), 1, 1)):
            with pytest.raises(NotImplementedError):
                DistributedB200Engine.aggregate(fake, B200DataFrame(t), PartitionSpec(by=["k"]), [fn(arg).alias("m")])
            with pytest.raises(NotImplementedError):
                DistributedB200Engine.aggregate(fake, B200DataFrame(t), None, [fn(arg).alias("m")])
