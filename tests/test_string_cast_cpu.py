"""Casts from strings (K13) without a GPU: the power-of-five table against Python integers, the parse routines
(run on the CPU through ``fb_debug_string_parse_host``) against pyarrow's own ``cast(safe=False)`` bit for bit on
every corpus of tests/_string_cast_corpus.py, the programs the compiler emits for a cast (run by the numpy machine
model over parse tables computed by the host export), the result cache, the error rule, string literal casts, the
targets that stay on the host, and the SQL type names of CAST."""
import os
import re

import numpy as np
import pyarrow as pa
import pytest
import torch

import _lookup_sim as lsim
import _string_cast_corpus as C
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.column import ColumnExpr, col, lit, to_sql, functions as ff
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table, expr_type

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the power-of-five table ----------------------------------------------------------------------------------
def _pow5_reference(q: int) -> int:
    """5^q with exactly 128 bits: truncated for q >= 0; floor(2^b / 5^-q) + 1, then truncated, for q < 0."""
    if q >= 0:
        p = 5 ** q
        return p << (128 - p.bit_length()) if p.bit_length() <= 128 else p >> (p.bit_length() - 128)
    p = 5 ** -q
    b = p.bit_length() + 127 if q >= -27 else 2 * p.bit_length() + 128
    c = (1 << b) // p + 1
    return c >> max(c.bit_length() - 128, 0)


def test_pow5_table_is_the_truncated_powers_of_five():
    text = open(os.path.join(ROOT, "fugue_b200", "csrc", "fb_pow5.inc")).read()
    rows = re.findall(r"\{0x([0-9A-F]{16})ull, 0x([0-9A-F]{16})ull\},\s*//\s*(-?\d+)", text)
    assert [int(q) for _, _, q in rows] == list(range(-342, 309))
    for hi, lo, q in rows:
        v = int(hi, 16) << 64 | int(lo, 16)
        assert v.bit_length() == 128 and v == _pow5_reference(int(q)), q
    # a positive power below 2^128 is exact: 5^q shifted, nothing lost
    assert all(_pow5_reference(q) == 5 ** q << (128 - (5 ** q).bit_length()) for q in range(0, 56))


def test_pow5_table_is_current():
    import subprocess
    import sys

    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_pow5.py"), "--check"], capture_output=True)
    assert r.returncode == 0, r.stdout


# ---- the parser against pyarrow ------------------------------------------------------------------------------
def _compare(strings, types, undecided_ok=False):
    """Host export against pyarrow: same accept / reject, same 8-byte word (NaN sign included); returns the
    number of undecided entries.  An undecided entry must be one pyarrow parses (the host resolves it)."""
    undecided = 0
    for tp in types:
        want, ok = C.expected(strings, tp)
        got, got_valid, status = C.host_parse(strings, tp)
        und = status == K.PARSE_UNDECIDED
        undecided += int(und.sum())
        assert ok[und].all(), (tp, [strings[i] for i in np.nonzero(und & ~ok)[0][:5]])
        decided = ~und
        bad = decided & (((status == K.PARSE_OK) != ok) | (ok & (got != want)))
        assert not bad.any(), (tp, [(strings[i], hex(int(want[i]) & (2 ** 64 - 1)), int(status[i]),
                                     hex(int(got[i]) & (2 ** 64 - 1))) for i in np.nonzero(bad)[0][:5]])
        assert (got_valid[decided] == (status[decided] == K.PARSE_OK)).all()
    if not undecided_ok:
        assert undecided == 0
    return undecided


def test_corners_every_target():
    _compare(C.CORNERS + C.int_corpus(), C.ALL_TYPES)


def test_nan_sign_and_float32_rounding():
    got, _, st = C.host_parse(["-nan", "nan", "3.4028235e38", "3.5e38", "-0"], pa.float32())
    assert (st == K.PARSE_OK).all()
    assert [int(x) & (2 ** 64 - 1) for x in got[:2]] == [0xFFF8000000000000, 0x7FF8000000000000]
    assert got[2:4].view(np.float64).tolist() == [float(np.finfo(np.float32).max), float("inf")]
    assert int(got[4]) & (2 ** 64 - 1) == 1 << 63


def test_null_entries_and_empty_dictionary():
    strings = ["1", None, "x", None, "2"]
    got, valid, st = C.host_parse(strings, pa.int64())
    assert st.tolist() == [K.PARSE_OK, K.PARSE_NULL, K.PARSE_INVALID, K.PARSE_NULL, K.PARSE_OK]
    assert valid.tolist() == [1, 0, 0, 0, 1] and got[[0, 4]].tolist() == [1, 2]
    got, valid, st = C.host_parse([], pa.float64())
    assert len(got) == len(valid) == len(st) == 0


def test_random_doubles():
    strings = C.random_doubles(1_000_000, 11)
    _compare(strings, [pa.float64()], undecided_ok=True)
    short = [s for s in strings if len(s.lstrip("-").replace(".", "").split("e")[0].lstrip("0")) <= 19]
    assert len(short) > 1_000_000
    assert _compare(short, [pa.float64()]) == 0  # at most 19 significant digits: never undecided


def test_random_doubles_as_float32():
    _compare(C.random_doubles(100_000, 12), [pa.float32()], undecided_ok=True)
    floats = np.random.default_rng(13).integers(0, 0x7F800000, 200_000).astype(np.uint32).view(np.float32)
    _compare([repr(float(f)) for f in floats] + ["%.9g" % f for f in floats], [pa.float32()])


def test_halfway_points_go_through_the_fallback_and_match(host_parse):
    before = ST.parse_fallbacks
    h64, h32 = C.halfway_corpus(400, 14), C.halfway_corpus(400, 15, f32=True)
    assert _compare(h64, [pa.float64()], undecided_ok=True) > 0
    assert _compare(h32, [pa.float32()], undecided_ok=True) > 0
    # the host resolves them: parse_table (with the host export standing in for the kernel) equals pyarrow
    for strings, tp in ((h64, pa.float64()), (h32, pa.float32())):
        d = pa.array(strings)
        r = ST._parse(d, torch.device("cpu"), tp)
        want, ok = C.expected(strings, tp)
        assert ok.all() and r.bad is None and r.valid is None
        assert (r.values.numpy() == want).all()
    assert ST.parse_fallbacks > before


def test_float_boundaries():
    _compare(C.boundary_floats(), [pa.float64(), pa.float32()], undecided_ok=True)


def test_every_date():
    _compare(C.all_dates(), [pa.date32(), pa.date64(), pa.timestamp("s")])


def test_random_timestamps():
    _compare(C.random_timestamps(50_000, 16), C.TS_TYPES + [pa.date32()])


def test_mutants():
    seeds = C.CORNERS + C.int_corpus() + C.random_timestamps(3000, 17) + C.random_doubles(1000, 18)[:3000]
    _compare(C.mutants(seeds, 40_000, 19), C.ALL_TYPES, undecided_ok=True)


def test_long_entries():
    strings = ["1" * 3000, "0" * 4000 + "1", "0." + "0" * 3000 + "1e3001", "1" + "0" * 2000 + "e-2000",
               "2024-01-02T03:04:05" + "0" * 2000, "0" * 3000 + "7"]
    _compare(strings, C.ALL_TYPES, undecided_ok=True)


# ---- the compiler --------------------------------------------------------------------------------------------
def _host_string_parse(offsets, data, valid, target):
    """``K.string_parse`` on CPU tensors, by the host export: the parse table of the compiler's tests."""
    out, out_valid, status = K.string_parse_host(offsets.numpy(), data.numpy(),
                                                 None if valid is None else valid.numpy(), target)
    bad = np.nonzero(status >= K.PARSE_INVALID)[0]
    return (torch.from_numpy(out.copy()), torch.from_numpy(out_valid.copy()), torch.from_numpy(status.copy()),
            int(bad[0]) if len(bad) else None)


@pytest.fixture
def host_parse(monkeypatch):
    from test_string_build_cpu import _oracle_evaluate  # string expressions over the dictionary, by the oracle

    monkeypatch.setattr(K, "string_parse", _host_string_parse)
    monkeypatch.setattr(ST, "evaluate", _oracle_evaluate)


def _table(entries, codes, row_valid=None, large=False):
    d = pa.array(entries, type=pa.large_string() if large else pa.string())
    n = len(codes)
    v = torch.arange(n, dtype=torch.int64)
    return B200Table(Schema("s:str,v:long"), [torch.tensor(codes, dtype=torch.int32), v],
                     [None if row_valid is None else torch.tensor(row_valid, dtype=torch.uint8), None], {"s": d})


def _run(t, e, out_type=K.T_I64):
    prog = X._Program(t)
    cls, _ = prog.compile(e, top=True)
    prog.output(torch.int64, True)
    cols = [t.columns[i] if isinstance(i, int) else prog.tables[i][0] for i in prog.cols]
    valid = [t.valid[i] if isinstance(i, int) else prog.tables[i][1] for i in prog.cols]
    types = [expr_type(t.schema.types[i]) if isinstance(i, int) else K.T_I64 for i in prog.cols]
    outs, outv = lsim.run(t.num_rows, [c.numpy() for c in cols], [None if m is None else m.numpy() for m in valid],
                          prog.ins, [out_type], col_types=types)
    return prog, cls, [int(x) if ok else None for x, ok in zip(outs[0].astype(np.uint64).view(np.int64), outv[0])]


def _want(values, tp):
    w, ok = C.expected(values, tp)
    return [int(x) if k else None for x, k in zip(w, ok)]


@pytest.mark.parametrize("large", [False, True])
def test_cast_of_a_column_compiles_to_a_lookup(host_parse, large):
    entries = ["12", "-3", None, "0x7f", "40"]
    codes = [0, 1, 2, 3, 4, 0, 4]
    t = _table(entries, codes, [1, 1, 1, 1, 1, 0, 1], large)
    prog, cls, got = _run(t, col("s").cast(pa.int8()))
    assert cls == "i"
    assert [i[0] for i in prog.ins] == [K.X_MOV, K.X_LOOKUP, K.X_OUT]
    assert got == [12, -3, None, 127, 40, None, 40]
    t = _table(["12", "-3", None, "1e2", "40"], codes, [1, 1, 1, 1, 1, 0, 1], large)
    prog, cls, got = _run(t, col("s").cast(pa.float64()) * 2 + col("v"))
    assert cls == "f"
    exp = [24.0, -5.0, None, 203.0, 84.0, None, 86.0]
    assert [None if g is None else float(np.int64(g).view(np.float64)) for g in got] == exp


def test_cast_of_a_string_expression(host_parse):
    entries = [" 12", "7 ", None, "  -4  ", "x"]
    t = _table(entries, [0, 1, 2, 3, 0, 3])
    prog, cls, got = _run(t, ff.trim(col("s")).cast("long"))
    assert any(i[0] == K.X_LOOKUP for i in prog.ins) and cls == "i"
    assert got == [12, 7, None, -4, 12, -4]
    with pytest.raises(ValueError, match="Failed to parse string: ' 12' as a scalar of type int64"):
        _run(t, col("s").cast("long"))  # Arrow refuses spaces: CAST(TRIM(s) AS long) is the idiom


def test_temporal_result_meets_its_literal(host_parse):
    import datetime

    entries = ["2024-01-01", "2023-12-31", "2024-02-29"]
    t = _table(entries, [0, 1, 2])
    _, cls, got = _run(t, col("s").cast("date") >= lit(datetime.date(2024, 1, 1)))
    assert got == [1, 0, 1]
    _, _, got = _run(t, col("s").cast(pa.timestamp("ms")) < lit(datetime.datetime(2024, 1, 1, 0, 0, 1)))
    assert got == [1, 1, 0]


def test_results_are_cached_per_dictionary(host_parse):
    t = _table(["1", "2", "3"], [0, 1, 2, 2])
    before = ST.parses
    _run(t, col("s").cast("int"))
    _run(t, col("s").cast("int") + 1)
    assert ST.parses == before + 1
    _run(t, col("s").cast("double"))
    assert ST.parses == before + 2
    t2 = _table(["1", "2", "3"], [0])
    _run(t2, col("s").cast("int"))  # another dictionary object: parsed again
    assert ST.parses == before + 3


def test_error_only_for_referenced_invalid_entries(host_parse):
    entries = ["1", "oops", "3", None]
    # entry 1 is not referenced by any valid row: a NULL row's code points at it
    t = _table(entries, [0, 2, 1, 3], [1, 1, 0, 1])
    _, _, got = _run(t, col("s").cast("int"))
    assert got == [1, 3, None, None]
    t = _table(entries, [0, 2, 1], [1, 1, 1])
    with pytest.raises(ValueError, match="Failed to parse string: 'oops' as a scalar of type int32"):
        _run(t, col("s").cast("int"))
    # a CASE does not shield the cast: every branch runs on every row
    with pytest.raises(ValueError):
        _run(t, ff.case([(col("v") > 5, col("s").cast("int"))], 0))
    # through a string expression: the entry after the expression is named
    with pytest.raises(ValueError, match="'OOPS'"):
        _run(t, ff.upper(col("s")).cast("int"))


def test_string_literal_casts_fold_on_the_host():
    t = _table(["1"], [0])
    for text, tp, want in [("12", pa.int64(), 12), ("0xff", pa.int8(), -1), ("1.5", pa.float64(), 1.5),
                           ("TRUE", pa.bool_(), True), ("2024-01-02", pa.date32(), 19724),
                           ("2024-01-02T00:00:01", pa.timestamp("ms"), 1704153601000)]:
        e = X.string_literal_cast(lit(text).cast(tp))
        assert e.value == want and e.as_type == tp, text
        prog = X._Program(t)
        prog.compile(lit(text).cast(tp))
        assert all(i[0] != K.X_LOOKUP for i in prog.ins)
    with pytest.raises(ValueError, match="Failed to parse string: 'x' as a scalar of type int64"):
        X.string_literal_cast(lit("x").cast("long"))


def test_targets_off_the_list_stay_on_the_host(host_parse):
    t = _table(["1"], [0])
    for tp in (pa.float16(), pa.decimal128(10, 2), pa.binary(), pa.time64("us"), pa.duration("s"),
               pa.list_(pa.int64())):
        with pytest.raises(NotImplementedError):
            X._Program(t).compile(col("s").cast(tp), top=True)
        with pytest.raises(NotImplementedError):
            X.string_literal_cast(lit("1").cast(tp))


def test_rejections_that_stay():
    t = _table(["1"], [0])
    with pytest.raises(NotImplementedError):  # a string function of a number
        X._Program(t).compile(ff.upper(col("s").cast(int)) == "A", top=True)
    with pytest.raises(NotImplementedError):  # string_codes is never handed a cast node
        X._Program(t).string_codes(ff.upper(col("s")).cast(int))


# ---- SQL -----------------------------------------------------------------------------------------------------
def _item(text: str) -> ColumnExpr:
    return _parse_select(text, "t", "SELECT " + text + " FROM t").columns[0]


@pytest.mark.parametrize("name,tp", [
    ("bigint", pa.int64()), ("BIGINT", pa.int64()), ("integer", pa.int32()), ("int", pa.int32()),
    ("smallint", pa.int16()), ("tinyint", pa.int8()), ("real", pa.float32()), ("double", pa.float64()),
    ("double precision", pa.float64()), ("varchar", pa.string()), ("text", pa.string()), ("boolean", pa.bool_()),
    ("bool", pa.bool_()), ("date", pa.date32()), ("timestamp", pa.timestamp("us")), ("datetime", pa.timestamp("us")),
    ("timestamp(ns)", pa.timestamp("ns")), ("timestamp(ns, UTC)", pa.timestamp("ns", "UTC")),
    ("timestamp(ms,Asia/Tokyo)", pa.timestamp("ms", "Asia/Tokyo")), ("timestamp(s, 'UTC')", pa.timestamp("s", "UTC")),
    ("long", pa.int64()), ("float", pa.float32()), ("str", pa.string()),
])
def test_sql_cast_type_names(name, tp):
    e = _item(f"CAST(s AS {name})")
    assert e.as_type == tp
    back = _item(to_sql(e))  # printer -> parser fixed point
    assert back.as_type == tp and to_sql(back) == to_sql(e)


def test_sql_cast_in_a_where_clause():
    q = _parse_select("*", "t WHERE CAST(TRIM(s) AS bigint) > 3 AND CAST(d AS timestamp(ns, UTC)) IS NOT NULL",
                      "SELECT * FROM t WHERE ...")
    assert q.where.fingerprint() == ((ff.trim(col("s")).cast(pa.int64()) > 3) &
                                     col("d").cast(pa.timestamp("ns", "UTC")).not_null()).fingerprint()
