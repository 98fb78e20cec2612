"""Casts from strings on the H100: the parse kernel (K13) entry for entry against the host export of the same
routines (which tests/test_string_cast_cpu.py checks against pyarrow) across the grid-stride bounds, and every
engine route that compiles a cast (select, filter, assign, aggregate argument and group key, SQL, ColumnMap,
alter_columns) against pyarrow's own cast, with the error rule and its exception types."""
import datetime

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import _string_cast_corpus as C
from test_dataframe_suite import ALTER_CASES
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import col, lit, functions as ff
from fugue_b200.dataframe import B200DataFrame, DataFrame, FugueDataFrameOperationError
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table

DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


def _kernel_equals_host(strings, types):
    offs, data, valid = C.layout(strings)
    d_offs = torch.from_numpy(offs).to(DEV)
    d_data = torch.from_numpy(data.copy() if len(data) else np.zeros(1, np.uint8)).to(DEV)
    d_valid = None if valid is None else torch.from_numpy(valid).to(DEV)
    for tp in types:
        target = ST.parse_target(tp)
        out, out_valid, status, first_bad = K.string_parse(d_offs, d_data, d_valid, target)
        h_out, h_valid, h_status = K.string_parse_host(offs, data, valid, target)
        assert np.array_equal(status.cpu().numpy(), h_status), tp
        assert np.array_equal(out_valid.cpu().numpy(), h_valid), tp
        assert np.array_equal(out.cpu().numpy(), h_out), tp
        bad = np.nonzero(h_status >= K.PARSE_INVALID)[0]
        assert first_bad == (int(bad[0]) if len(bad) else None), tp


def test_kernel_equals_host_export_on_every_corpus():
    seeds = C.CORNERS + C.int_corpus() + C.random_timestamps(3000, 1)
    strings = (C.CORNERS + C.int_corpus() + C.boundary_floats() + C.random_doubles(50_000, 2) +
               C.halfway_corpus(100, 3) + C.halfway_corpus(100, 4, f32=True) + C.random_timestamps(50_000, 5) +
               C.mutants(seeds, 50_000, 6) + ["7" * 3000, "0." + "0" * 4000 + "5e4001", "2024-01-02" + " " * 2000])
    with_nulls = [None if i % 97 == 13 else s for i, s in enumerate(strings)]
    _kernel_equals_host(with_nulls, C.ALL_TYPES)


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 3_000_000])
def test_kernel_across_grid_stride_bounds(n):
    rng = np.random.default_rng(n)
    pool = C.CORNERS + C.random_doubles(2000, 7)[:2000] + C.random_timestamps(2000, 8) + [None]
    strings = [pool[i] for i in rng.integers(0, len(pool), n)] if n else []
    _kernel_equals_host(strings, [pa.int32(), pa.float64(), pa.float32(), pa.timestamp("us"),
                                  pa.timestamp("ns", "UTC"), pa.date32(), pa.bool_()])


def test_undecided_entries_are_resolved_on_the_host():
    h = C.halfway_corpus(200, 9)
    before = ST.parse_fallbacks
    r = ST.parse_table(pa.array(h), DEV, pa.float64())
    want, ok = C.expected(h, pa.float64())
    assert ok.all() and r.bad is None and np.array_equal(r.values.cpu().numpy(), want)
    assert ST.parse_fallbacks > before


# ---- engine routes --------------------------------------------------------------------------------------------
def _frame(rng, n, entries, large=False, null_rows=0.1):
    """A frame of string column s over ``entries`` (with NULL rows), a group key k and a row id."""
    codes = rng.integers(0, len(entries), n)
    mask = rng.random(n) < null_rows
    typ = pa.large_string() if large else pa.string()
    s = pa.array([None if m else entries[c] for c, m in zip(codes, mask)], type=typ)
    tbl = pa.table({"rid": np.arange(n), "k": rng.integers(0, 7, n), "s": s})
    return B200DataFrame(B200Table.from_arrow(tbl, DEV)), tbl


def _cast(arr, tp):
    return pc.cast(arr, tp, safe=False)


ENTRY_SETS = {
    pa.int64(): ["12", "-7", "0x10", "007", "9223372036854775807", "-0", None],
    pa.int16(): ["32767", "-32768", "0xffff", "5"],
    pa.uint32(): ["4294967295", "0", "0xFFFFFFFF", "17"],
    pa.float64(): ["1.5", "-2.25e3", "inf", "-nan", "4.9e-324", "0.1000000000000000055511151231257827", "1e400"],
    pa.float32(): ["3.4028235e38", "1e-5", "-0", "-inf", "16777217"],
    pa.bool_(): ["true", "FALSE", "1", "0", None],
    pa.date32(): ["2024-01-01", "1900-03-01", "0001-01-01", "9999-12-31", "2024-02-29"],
    pa.timestamp("us"): ["2024-01-02T03:04:05.123456", "1969-12-31 23:59:59", "2024-01-02", "2024-01-02T03"],
    pa.timestamp("ns", "UTC"): ["2024-01-02T03:04:05.123456789Z", "2024-01-02T03:04+05:30", "1999-12-31T23-0100"],
    pa.date64(): ["2024-01-01", "1970-01-02"],
}


@pytest.mark.parametrize("large", [False, True])
@pytest.mark.parametrize("tp", list(ENTRY_SETS), ids=[str(t) for t in ENTRY_SETS])
def test_select_assign_and_column_map(e, tp, large):
    rng = np.random.default_rng(10)
    df, tbl = _frame(rng, 5000, ENTRY_SETS[tp], large)
    want = _cast(tbl.column("s"), tp).combine_chunks()
    got = fa.select(df, col("rid"), col("s").cast(tp).alias("x"), engine=e, as_fugue=True).as_arrow()
    assert got.schema.field("x").type == tp
    assert C.words(got.column("x").combine_chunks()).tolist() == C.words(want).tolist()
    assert got.column("x").is_valid().to_pylist() == want.is_valid().to_pylist()
    got = fa.assign(df, x=col("s").cast(tp), engine=e, as_fugue=True).as_arrow()
    assert C.words(got.column("x").combine_chunks()).tolist() == C.words(want).tolist()
    if tp == pa.float64():
        rid = df.native.columns[0]
        got = fa.transform(df, ColumnMap("rid", col("s").cast(tp).alias("x")), schema="rid:long,x:double",
                           partition=PartitionSpec(by="k", presort="rid"), engine=e, as_fugue=True).as_arrow()
        order = np.argsort(got.column("rid").to_numpy())
        assert C.words(got.column("x").combine_chunks().take(order)).tolist() == C.words(want).tolist()
        assert int(rid.shape[0]) == got.num_rows


def test_filter_aggregate_and_group_key(e):
    rng = np.random.default_rng(11)
    entries = ["2024-01-01", "2023-12-31", "2024-06-30", "1999-01-01"]
    df, tbl = _frame(rng, 20_000, entries)
    got = fa.filter(df, col("s").cast("date") >= lit(datetime.date(2024, 1, 1)), engine=e, as_fugue=True).as_arrow()
    d = _cast(tbl.column("s"), pa.date32())
    keep = pc.fill_null(pc.greater_equal(d, pa.scalar(datetime.date(2024, 1, 1))), False)
    assert got.column("rid").to_pylist() == tbl.filter(keep).column("rid").to_pylist()
    nums = ["1.5", "2", "-0.25", "1e3"]
    df, tbl = _frame(rng, 20_000, nums)
    got = fa.aggregate(df, "k", x=ff.sum(col("s").cast(float)), engine=e, as_fugue=True).as_arrow()
    v = _cast(tbl.column("s"), pa.float64()).to_pylist()
    want = {}
    for k, x in zip(tbl.column("k").to_pylist(), v):
        if x is not None:
            want[k] = want.get(k, 0.0) + x
    assert dict(zip(got.column("k").to_pylist(), got.column("x").to_pylist())) == pytest.approx(want)
    ints = ["1", "2", "02", "3"]
    df, tbl = _frame(rng, 20_000, ints)
    got = fa.raw_sql("SELECT CAST(s AS int) AS c, COUNT(*) AS n FROM", df, "GROUP BY CAST(s AS int)", engine=e,
                     as_fugue=True).as_arrow()
    # the group keys of a SELECT are its columns without their casts (SelectColumns.group_keys): one group per
    # string, whose key is then cast, so "2" and "02" are two groups with c = 2
    strs = tbl.column("s").to_pylist()
    want = [(None if v is None else int(v), strs.count(v)) for v in set(strs)]
    assert sorted(zip(got.column("c").to_pylist(), got.column("n").to_pylist()), key=str) == sorted(want, key=str)


def test_sql_on_a_csv_read_as_text(e, tmp_path):
    rng = np.random.default_rng(12)
    n = 10_000
    ts = ["2024-01-02 03:04:05", "2024-01-02T03:04:05.5", "2023-07-01"]
    rows = [(ts[i], f"{x:.6g}") for i, x in zip(rng.integers(0, 3, n), rng.standard_normal(n))]
    path = str(tmp_path / "t.csv")
    with open(path, "w") as f:
        f.write("s,v\n" + "".join(f"{a},{b}\n" for a, b in rows))
    df = fa.load(path, header=True, engine=e, as_fugue=True)
    assert [str(t) for t in df.schema.types] == ["string", "string"]
    got = fa.raw_sql("SELECT CAST(s AS timestamp) AS t, SUM(CAST(v AS double)) AS x FROM", df,
                     "GROUP BY CAST(s AS timestamp)", engine=e, as_fugue=True).as_arrow()
    t = _cast(pa.array([r[0] for r in rows]), pa.timestamp("us")).to_pylist()
    v = _cast(pa.array([r[1] for r in rows]), pa.float64()).to_pylist()
    want = {}
    for a, b in zip(t, v):
        want[a] = want.get(a, 0.0) + b
    assert dict(zip(got.column("t").to_pylist(), got.column("x").to_pylist())) == pytest.approx(want)
    with pytest.raises(ValueError, match="as a scalar of type date32"):  # Arrow refuses a time part in a date
        fa.raw_sql("SELECT COUNT(*) AS n FROM", df, "WHERE CAST(s AS date) >= DATE '2024-01-01'", engine=e)
    got = fa.raw_sql("SELECT COUNT(*) AS n FROM", df, "WHERE CAST(s AS timestamp) >= TIMESTAMP '2024-01-01 00:00:00'",
                     engine=e, as_fugue=True).as_arrow()
    assert got.column("n").to_pylist() == [sum(r[0] >= "2024" for r in rows)]


def test_trimmed_cast_and_the_error_rule(e):
    rng = np.random.default_rng(13)
    df, tbl = _frame(rng, 3000, [" 1", "2 ", " 30 "])
    got = fa.select(df, ff.trim(col("s")).cast("long").alias("x"), engine=e, as_fugue=True).as_arrow()
    assert got.column("x").to_pylist() == _cast(pc.utf8_trim_whitespace(tbl.column("s")), pa.int64()).to_pylist()
    with pytest.raises(ValueError, match=r"Failed to parse string: '( 1|2 | 30 )' as a scalar of type int64"):
        fa.select(df, col("s").cast("long").alias("x"), engine=e)
    # an invalid entry that a filter leaves unreferenced raises nothing
    df, tbl = _frame(rng, 3000, ["1", "2", "oops"], null_rows=0.0)
    kept = fa.filter(df, col("s") != "oops", engine=e, as_fugue=True)
    assert kept.native.dictionaries["s"].to_pylist().count("oops") == 1
    got = fa.select(kept, col("s").cast("int").alias("x"), engine=e, as_fugue=True).as_arrow()
    assert sorted(set(got.column("x").to_pylist())) == [1, 2]
    with pytest.raises(ValueError, match="'oops'"):
        fa.select(df, col("s").cast("int").alias("x"), engine=e)
    with pytest.raises(ValueError):  # a CASE does not shield the cast
        fa.select(df, ff.case([(col("s") == "oops", 0)], col("s").cast("int")).alias("x"), engine=e)
    with pytest.raises(FugueDataFrameOperationError):
        fa.alter_columns(df, "s:int")


ALTER_STR = [c for c in ALTER_CASES if c[0] == "a:str,b:str"]


@pytest.mark.parametrize("schema,rows,alter,after,accepted", ALTER_STR, ids=[c[2] for c in ALTER_STR])
def test_alter_columns_on_device_frames(e, monkeypatch, schema, rows, alter, after, accepted):
    calls = []
    base = DataFrame.alter_columns
    monkeypatch.setattr(DataFrame, "alter_columns", lambda self, c: calls.append(c) or base(self, c))
    df = e.to_df(fa.as_fugue_df(rows, schema).as_arrow())
    assert isinstance(df, B200DataFrame)
    out = df.alter_columns(alter)
    assert isinstance(out, B200DataFrame) and calls == []
    assert str(out.schema) == after
    assert out.as_array(type_safe=True) in accepted


def test_alter_columns_keeps_the_host_path_for_other_targets(e, monkeypatch):
    calls = []
    base = DataFrame.alter_columns
    monkeypatch.setattr(DataFrame, "alter_columns", lambda self, c: calls.append(c) or base(self, c))
    df = e.to_df(pa.table({"a": ["1.5", "2"]}))
    out = df.alter_columns("a:float16")
    assert calls == ["a:float16"] and out.as_arrow().column("a").type == pa.float16()
