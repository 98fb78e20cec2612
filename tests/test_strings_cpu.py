"""LIKE, LENGTH and string MIN / MAX without a GPU: the builders, typing, SQL text and parser, the rejections,
the LIKE tokenizer, the K8 programs the compiler emits (run by the numpy machine model, tests/_expr_sim.py, with
FB_X_LOOKUP from tests/_lookup_sim.py) against oracle/strings.py and oracle/expressions.py, the model's lookup itself,
and the multi-GPU rejection of string MIN / MAX."""
import random
import types

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest
import torch

import _lookup_sim as lsim
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.column import ColumnExpr, Kind, col, lit, to_sql, functions as ff
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table, expr_type
from oracle import expressions as ox
from oracle import strings as ostr

# characters of 1, 2, 3 and 4 UTF-8 bytes, and the pattern's special characters as data
ALPHABET = ["a", "b", "c", "%", "_", "!", "\\", "é", "ß", "€", "中", "😀", "𝄞"]


def _parse_where(text: str) -> ColumnExpr:
    return _parse_select("*", "t WHERE " + text, "SELECT * FROM t WHERE " + text).where


# ---- builders, typing, SQL text ------------------------------------------------------------------------
def test_builders_and_types():
    sch = Schema("s:str,v:long")
    e = col("s").like("a%")
    assert e.kind == Kind.CALL and e.func == "LIKE" and e.infer_type(sch) == pa.bool_()
    assert col("s").like(lit("a%")).fingerprint() == e.fingerprint()
    n = ff.length(col("s"))
    assert n.kind == Kind.CALL and n.func == "LENGTH" and n.infer_type(sch) == pa.int64()
    assert ff.length("s").fingerprint() == n.fingerprint()
    assert (~e).infer_type(sch) == pa.bool_()


@pytest.mark.parametrize("expr,text", [
    (col("s").like("a%"), "s LIKE 'a%'"),
    (col("s").like("a!%", escape="!"), "s LIKE 'a!%' ESCAPE '!'"),
    (ff.length(col("s")), "LENGTH(s)"),
    (~col("s").like("_b%"), "NOT (s LIKE '_b%')"),
    (col("s").like("it's"), "s LIKE 'it\\'s'"),
    (col("s").like("a\\%", escape="\\"), "s LIKE 'a\\\\%' ESCAPE '\\\\'"),
])
def test_printer_parser_round_trip(expr, text):
    assert to_sql(expr) == text
    assert _parse_where(text).fingerprint() == expr.fingerprint()


def test_parser_forms():
    assert _parse_where("s NOT LIKE 'a!_%' ESCAPE '!'").fingerprint() == (~col("s").like("a!_%", "!")).fingerprint()
    assert _parse_where("s LIKE 'x' AND v > 0").fingerprint() == (col("s").like("x") & (col("v") > 0)).fingerprint()
    assert _parse_where("LENGTH(s) * 2 > 3").fingerprint() == (ff.length(col("s")) * 2 > 3).fingerprint()
    st = _parse_select("LENGTH(s) AS n, MAX(s) AS m", "t GROUP BY v", "")
    assert [c.fingerprint() for c in st.columns] == [ff.length(col("s")).alias("n").fingerprint(),
                                                   ff.max(col("s")).alias("m").fingerprint()]


def test_builder_rejections():
    with pytest.raises(NotImplementedError):
        col("s").like(col("p"))
    with pytest.raises(NotImplementedError):
        _parse_where("s LIKE p")
    with pytest.raises(ValueError):
        col("s").like("ab!", escape="!")
    with pytest.raises(ValueError):
        _parse_where("s LIKE 'ab!' ESCAPE '!'")
    with pytest.raises(ValueError):
        col("s").like("a", escape="!!")
    col("s").like("ab!!", escape="!")  # an escaped escape character is complete


# ---- the LIKE tokenizer -----------------------------------------------------------------------------------
def test_like_tokens():
    A, O = K.LIKE_ANY, K.LIKE_ONE
    assert ST.like_tokens("", None) == []
    assert ST.like_tokens("%%", None) == [A]
    assert ST.like_tokens("a%%_%", None) == [97, A, O, A]
    assert ST.like_tokens("é_", None) == [0xC3, 0xA9, O]
    assert ST.like_tokens("!%!_!!%", "!") == [37, 95, 33, A]
    assert ST.like_tokens("\\%", None) == [92, A]  # no default escape character
    with pytest.raises(ValueError):
        ST.like_tokens("a!", "!")
    ST.like_tokens("a" * K.LIKE_MAX_TOKENS, None)
    with pytest.raises(NotImplementedError):
        ST.like_tokens("a" * (K.LIKE_MAX_TOKENS + 1), None)


# ---- the oracle, pinned against pyarrow ------------------------------------------------------------------
def test_oracle_against_pyarrow():
    rng = random.Random(7)
    values = ["".join(rng.choice(ALPHABET[:4] + ALPHABET[7:]) for _ in range(rng.randint(0, 6))) for _ in range(300)]
    values += ["", "%", "_", None]
    arr = pa.array(values, type=pa.string())
    assert pc.utf8_length(arr).to_pylist() == [ostr.length(v) for v in values]
    pats = ["", "%", "%%", "_", "a%", "%a", "%é%", "_b_", "a%c", "%€_%", "%%b%%", "中%😀"]
    pats += ["".join(rng.choice(["a", "b", "é", "%", "_", "😀"]) for _ in range(rng.randint(1, 5))) for _ in range(40)]
    for p in pats:  # no backslash: pyarrow's default escape character then plays no part
        assert pc.match_like(arr, p).to_pylist() == [ostr.like(v, p) for v in values], p


# ---- the compiler and the machine model ------------------------------------------------------------------
def _entry_tables(monkeypatch):
    """Per-entry tables from the oracle instead of the device kernels, as CPU tensors."""

    def valid_of(d):
        return None if d.null_count == 0 else torch.tensor([v is not None for v in d.to_pylist()], dtype=torch.uint8)

    def like_table(d, device, pattern, escape):
        return torch.tensor([bool(ostr.like(v, pattern, escape)) for v in d.to_pylist()], dtype=torch.int64), valid_of(d)

    def length_table(d, device):
        return torch.tensor([ostr.length(v) or 0 for v in d.to_pylist()], dtype=torch.int64), valid_of(d)

    monkeypatch.setattr(ST, "like_table", like_table)
    monkeypatch.setattr(ST, "length_table", length_table)


def _random_table(rng: np.random.Generator, n: int, ndict: int, null_entries: bool, dict_type=pa.string()):
    words = set()
    while len(words) < ndict:
        k = int(rng.integers(0, 7))
        words.add("".join(ALPHABET[int(i)] for i in rng.integers(0, len(ALPHABET), k)))
    entries = sorted(words, key=lambda _: rng.random())
    if null_entries:
        entries[int(rng.integers(0, ndict))] = None
    d = pa.array(entries, type=dict_type)
    codes = rng.integers(0, ndict, n).astype(np.int32)
    valid = (rng.random(n) > 0.2).astype(np.uint8)
    matchy = [i for i, w in enumerate(entries) if w is not None and w.startswith("a")]
    if matchy:  # NULL rows whose stored code is an entry that matches
        codes[valid == 0] = matchy[0]
    v = rng.integers(-5, 5, n).astype(np.int64)
    t = B200Table(Schema("s:str,v:long"), [torch.from_numpy(codes), torch.from_numpy(v)],
                  [torch.from_numpy(valid), None], {"s": d})
    pdf = pd.DataFrame({"s": pd.array([entries[c] if m else None for c, m in zip(codes, valid)], dtype="string"),
                        "v": v})
    return t, pdf


def _run_model(t: B200Table, e: ColumnExpr):
    prog = X._Program(t)
    cls, nullable = prog.compile(e, top=True)
    tp = {"b": pa.bool_(), "i": pa.int64()}[cls]
    prog.output(torch.uint8 if cls == "b" else torch.int64, True)
    cols = [t.columns[i] if isinstance(i, int) else prog.tables[i][0] for i in prog.cols]
    valid = [t.valid[i] if isinstance(i, int) else prog.tables[i][1] for i in prog.cols]
    types = [expr_type(t.schema.types[i]) if isinstance(i, int) else K.T_I64 for i in prog.cols]
    outs, outv = lsim.run(t.num_rows, [c.numpy() for c in cols], [None if m is None else m.numpy() for m in valid],
                         prog.ins, [K.T_U8 if cls == "b" else K.T_I64], col_types=types)
    return prog, [None if not ok else (bool(x) if tp == pa.bool_() else int(x)) for x, ok in zip(outs[0], outv[0])]


def _expected(pdf: pd.DataFrame, e: ColumnExpr):
    df2, (e2,), _ = ostr.lower(pdf, [e])
    v = ox.evaluate(e2, df2)
    return [None if x is pd.NA else (bool(x) if isinstance(x, (bool, np.bool_)) else int(x)) for x in v]


PATTERNS = [("", None), ("%", None), ("%%", None), ("_", None), ("a%", None), ("%a", None), ("%a%b%", None),
            ("_é%", None), ("%€", None), ("%😀_", None), ("__", None), ("a_%_c", None), ("%中%𝄞%", None),
            ("!%%", "!"), ("%!%", "!"), ("!_%", "!"), ("%!!%", "!"), ("a!_b", "!"), ("%\\%", None),
            ("\\%%", "\\"), ("%_%_%", None), ("%%%", None)]


def test_compiler_emits_lookup_programs(monkeypatch):
    _entry_tables(monkeypatch)
    t, _ = _random_table(np.random.default_rng(0), 100, 20, False)
    prog, _ = _run_model(t, col("s").like("a%"))
    ops = [i[0] for i in prog.ins]
    assert ops[:2] == [K.X_MOV, K.X_LOOKUP] and prog.ins[1][1] == K.XK_COL and prog.ins[1][4] == 20
    prog, _ = _run_model(t, (col("s").like("a%") & (col("v") > 0)) | (ff.length(col("s")) * 2 > 3))
    assert [i[0] for i in prog.ins].count(K.X_LOOKUP) == 2 and len(prog.cols) == 4
    prog, _ = _run_model(t, col("s").like("a%") | ~col("s").like("a%"))  # one table for one (column, pattern)
    assert len(prog.cols) == 2


@pytest.mark.parametrize("seed", range(6))
def test_model_matches_oracle(monkeypatch, seed):
    _entry_tables(monkeypatch)
    rng = np.random.default_rng(seed)
    t, pdf = _random_table(rng, 3000, int(rng.integers(1, 60)), null_entries=seed % 2 == 1,
                           dict_type=pa.large_string() if seed % 3 == 0 else pa.string())
    exprs = [ff.length(col("s")), ff.length(col("s")) * 2 + col("v"), ff.length(col("s")) > 2,
             (col("v") * 2 + 1) * (ff.length(col("s")) - 1),  # a temporary held across the lookup
             ((col("v") > 0) | (col("v") < -3)) & (col("s").like("%a%") | (ff.length(col("s")) * col("v") > 4))]
    for p, esc in PATTERNS:
        e = col("s").like(p, esc)
        exprs += [e, ~e, e & (col("v") > 0), (col("v") < 0) | e]
    for e in exprs:
        _, got = _run_model(t, e)
        assert got == _expected(pdf, e), str(e)


def test_model_lookup():
    """FB_X_LOOKUP in the model: the entry's value and validity; NULL for a NULL accumulator, an entry number past
    the table or a negative code read as an unsigned entry number, and for any entry of an empty table."""
    acc = np.array([0, 2, 1, 3, (1 << 64) - 1, 1], dtype=np.uint64)
    accv = np.array([1, 1, 1, 1, 1, 0], dtype=bool)
    table = np.array([10, 20, 30], dtype=np.uint64)
    v, m = lsim.lookup(acc, accv, table, np.array([1, 0, 1], dtype=np.uint8), 3)
    assert v.tolist() == [10, 30, 20, 0, 0, 0] and m.tolist() == [True, True, False, False, False, False]
    v, m = lsim.lookup(acc, accv, table, None, 3)
    assert m.tolist() == [True, True, True, False, False, False]
    v, m = lsim.lookup(acc, accv, np.zeros(0, dtype=np.uint64), None, 0)
    assert not m.any() and not v.any()


def test_compiler_rejections(monkeypatch):
    _entry_tables(monkeypatch)
    t, _ = _random_table(np.random.default_rng(1), 10, 5, False)
    for e in [col("v").like("a%"), ff.length(col("v")), ff.length(lit("abc")), col("s").cast(str).like("a"),
              ColumnExpr(Kind.CALL, "LIKE", [col("s"), col("s")]), ColumnExpr(Kind.CALL, "UPPER", [col("s")]),
              col("s") < "b"]:
        with pytest.raises(NotImplementedError):
            X._Program(t).compile(e, top=True)


# ---- multi-GPU: string MIN / MAX stays unsupported ------------------------------------------------------
def test_distributed_string_min_max_raises():
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.dist import DistributedB200Engine
    from fugue_b200.partition import PartitionSpec

    t = B200Table(Schema("k:long,s:str"), [torch.tensor([1, 2]), torch.tensor([0, 1], dtype=torch.int32)], None,
                  {"s": pa.array(["x", "y"])})
    fake = types.SimpleNamespace(_world=2, to_df=lambda df: df)
    for fn in (ff.min, ff.max):
        with pytest.raises(NotImplementedError):
            DistributedB200Engine.aggregate(fake, B200DataFrame(t), PartitionSpec(by=["k"]), [fn(col("s")).alias("m")])
        with pytest.raises(NotImplementedError):
            DistributedB200Engine.aggregate(fake, B200DataFrame(t), None, [fn(col("s")).alias("m")])
