"""Casts to strings on the H100: the format kernel (K14) byte for byte against the host export of the same routines
(which tests/test_value_format_cpu.py checks against CPython and pyarrow), every route of a cast to string on every
storage type against ``ArrowDataFrame.alter_columns``, the dictionaries it builds, and casts inside expressions."""
import collections

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import col, functions as ff
from fugue_b200.dataframe import ArrowDataFrame
from fugue_b200.partition import PartitionSpec

DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


@pytest.mark.parametrize("kind", ["f64", "i64", "u64", "date32", "date64", "ts_s", "ts_ms", "ts_us", "ts_ns"])
def test_kernel_equals_host_export(kind):
    rng = np.random.default_rng(20)
    n = 10_000_000
    words = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64, endpoint=True)
    code = {"f64": K.FMT_F64, "i64": K.FMT_I64, "u64": K.FMT_U64, "date32": K.FMT_DATE32, "date64": K.FMT_DATE64,
            "ts_s": K.FMT_TS + K.TU_S, "ts_ms": K.FMT_TS + K.TU_MS + K.FMT_TS_FRAC,
            "ts_us": K.FMT_TS + K.TU_US + K.FMT_TS_FRAC, "ts_ns": K.FMT_TS + K.TU_NS + K.FMT_TS_FRAC}[kind]
    if kind == "date32":
        words = (words >> 32).astype(np.int64)
    valid = (rng.random(n) > 0.05).astype(np.uint8)
    offs, data = K.value_format(torch.from_numpy(words).to(DEV), torch.from_numpy(valid).to(DEV), code)
    h_offs, h_data = K.value_format_host(words, valid, code)
    assert np.array_equal(offs.cpu().numpy(), h_offs)
    assert np.array_equal(data.cpu().numpy()[:h_offs[-1]], h_data[:h_offs[-1]])


def _table(n=3000):
    """Every storage type a cast to string formats, with NULLs and edge values."""
    rng = np.random.default_rng(21)
    mask = rng.random(n) < 0.1
    cols = {}
    for name, tp in [("i8", pa.int8()), ("i16", pa.int16()), ("i32", pa.int32()), ("i64", pa.int64()),
                     ("u8", pa.uint8()), ("u16", pa.uint16()), ("u32", pa.uint32()), ("u64", pa.uint64())]:
        info = np.iinfo(tp.to_pandas_dtype())
        v = rng.integers(info.min, info.max, n, dtype=tp.to_pandas_dtype(), endpoint=True)
        v[:2] = [info.min, info.max]
        cols[name] = pa.array(v, tp, mask=mask)
    f = rng.standard_normal(n) * 10.0 ** rng.integers(-20, 20, n)
    f[:6] = [0.0, -0.0, np.nan, np.inf, -np.inf, 0.1]
    f[6] = np.frombuffer(np.uint64(0xFFF8000000000123).tobytes(), np.float64)[0]  # a NaN with sign and payload
    for name, tp in [("f16", pa.float16()), ("f32", pa.float32()), ("f64", pa.float64())]:
        cols[name] = pa.array(f.astype(tp.to_pandas_dtype()), tp, mask=mask)
    cols["b"] = pa.array(rng.random(n) < 0.5, pa.bool_(), mask=mask)
    days = rng.integers(-800_000, 3_000_000, n)
    cols["d32"] = pa.array(days.astype(np.int32), pa.int32(), mask=mask).view(pa.date32())
    cols["d64"] = pa.array(days * 86_400_000 + rng.integers(0, 86_400_000, n) * (np.arange(n) % 2),
                           pa.int64(), mask=mask).view(pa.date64())
    for unit, per in [("s", 1), ("ms", 1000), ("us", 10 ** 6), ("ns", 10 ** 9)]:
        secs = rng.integers(-2_000_000_000, 4_000_000_000, n)
        whole = pa.array(secs * per, pa.int64(), mask=mask)
        frac = pa.array(secs * per + rng.integers(0, per, n), pa.int64(), mask=mask)
        cols[f"t{unit}"] = frac.view(pa.timestamp(unit))
        cols[f"w{unit}"] = whole.view(pa.timestamp(unit))
        cols[f"z{unit}"] = frac.view(pa.timestamp(unit, "UTC"))
    cols["rid"] = pa.array(np.arange(n))
    return pa.table(cols)


def _host_text(tbl: pa.Table, name: str):
    return ArrowDataFrame(tbl.select([name])).alter_columns(f"{name}:str").as_arrow().column(0).to_pylist()


def test_every_route_on_every_type(e):
    tbl = _table()
    df = e.to_df(tbl)
    names = [n for n in tbl.column_names if n != "rid"]
    want = {n: _host_text(tbl, n) for n in names}
    got = fa.select(df, *[col(n).cast(str) for n in names], engine=e, as_fugue=True).as_arrow()
    for n in names:
        assert got.column(n).to_pylist() == want[n], n
    alt = fa.alter_columns(df, ",".join(f"{n}:str" for n in names), as_fugue=True)
    assert type(alt).__name__ == "B200DataFrame"
    for n in names:
        assert alt.as_arrow().column(n).to_pylist() == want[n], n
    got = fa.assign(df, x=col("f32").cast(str), engine=e, as_fugue=True).as_arrow()
    assert got.column("x").to_pylist() == want["f32"]
    got = fa.filter(df, col("i64").cast(str) == want["i64"][5], engine=e, as_fugue=True).as_arrow()
    assert got.column("rid").to_pylist() == [i for i, s in enumerate(want["i64"]) if s == want["i64"][5]]
    got = fa.raw_sql("SELECT rid, CAST(d32 AS STRING) AS s, CAST(tus AS VARCHAR) AS t FROM", df, engine=e,
                     as_fugue=True).as_arrow()
    assert got.column("s").to_pylist() == want["d32"] and got.column("t").to_pylist() == want["tus"]
    got = fa.transform(df, ColumnMap("rid", col("f64").cast(str).alias("x")), schema="rid:long,x:str",
                       partition=PartitionSpec(by="b", presort="rid"), engine=e, as_fugue=True).as_arrow()
    assert dict(zip(got.column("rid").to_pylist(), got.column("x").to_pylist())) == dict(enumerate(want["f64"]))
    got = fa.aggregate(df, "b", m=ff.max(col("i32").cast(str)), engine=e, as_fugue=True).as_arrow()
    exp = {}
    for b, s in zip(tbl.column("b").to_pylist(), want["i32"]):
        exp.setdefault(b, None)
        if s is not None:
            exp[b] = s if exp[b] is None else max(exp[b], s)
    assert dict(zip(got.column("b").to_pylist(), got.column("m").to_pylist())) == exp


def test_dictionaries_are_distinct():
    f = torch.tensor([0.0, -0.0, float("nan"), -float("nan"), 0.0, 1.0], dtype=torch.float64, device=DEV)
    f[3] = torch.tensor([0x7FF0000000000001], dtype=torch.int64).view(torch.float64)[0].to(DEV)
    codes, _, d = ST.format_values(f, None, pa.float64(), DEV)
    entries = d.to_pylist()
    assert sorted(entries) == sorted(["0.0", "-0.0", "nan", "1.0"]) and len(entries) == len(set(entries))
    assert [entries[c] for c in codes.tolist()] == ["0.0", "-0.0", "nan", "nan", "0.0", "1.0"]


def test_time_zones(e):
    tbl = pa.table({"t": pa.array([0, 1_700_000_000_000_000], pa.int64()).view(pa.timestamp("us", "Asia/Tokyo"))})
    df = e.to_df(tbl)
    with pytest.raises(NotImplementedError):
        fa.select(df, col("t").cast(str), engine=e)
    got = fa.alter_columns(df, "t:str", as_fugue=True).as_arrow().column(0).to_pylist()
    assert got == _host_text(tbl, "t")


def test_casts_inside_expressions(e):
    rng = np.random.default_rng(22)
    n = 50_000
    k = rng.integers(-500, 20_000, n)
    t = rng.integers(0, 2_000_000_000_000_000, n)
    tbl = pa.table({"id": np.arange(n), "k": k, "t": pa.array(t, pa.int64()).view(pa.timestamp("us"))})
    df = e.to_df(tbl)
    ks = [str(x) for x in k.tolist()]
    got = fa.raw_sql("SELECT CAST(k AS STRING) AS s, COUNT(*) AS n FROM", df, "GROUP BY CAST(k AS STRING)",
                     engine=e, as_fugue=True).as_arrow()
    assert dict(zip(got.column("s").to_pylist(), got.column("n").to_pylist())) == collections.Counter(ks)
    got = fa.raw_sql("SELECT id FROM", df, "WHERE CAST(k AS STRING) LIKE '12%'", engine=e, as_fugue=True).as_arrow()
    assert got.column("id").to_pylist() == [i for i, s in enumerate(ks) if s.startswith("12")]
    got = fa.select(df, col("id"), ff.concat(col("id").cast(str), "-x").alias("c"),
                    ff.length(col("k").cast(str)).alias("n"), engine=e, as_fugue=True).as_arrow()
    assert got.column("c").to_pylist() == [f"{i}-x" for i in range(n)]
    assert got.column("n").to_pylist() == [len(s) for s in ks]
    got = fa.raw_sql("SELECT MIN(CAST(k AS STRING)) AS lo, MAX(CAST(k AS STRING)) AS hi FROM", df, engine=e,
                     as_fugue=True).as_arrow()
    assert (got.column("lo")[0].as_py(), got.column("hi")[0].as_py()) == (min(ks), max(ks))
    s = fa.select(df, col("t"), col("t").cast(str).alias("s"), engine=e, as_fugue=True)
    back = fa.select(s, col("t"), col("s").cast(pa.timestamp("us")).alias("b"), engine=e, as_fugue=True).as_arrow()
    assert back.column("b").to_pylist() == back.column("t").to_pylist()
    got = fa.select(df, ff.trim(col("t").cast(str)).cast(pa.timestamp("us")).alias("b"), engine=e,
                    as_fugue=True).as_arrow()
    assert got.column("b").to_pylist() == tbl.column("t").to_pylist()


def test_like_on_a_cast_uploads_nothing(e):
    df = e.to_df(pa.table({"k": np.arange(100_000)}))
    before = ST.uploads
    got = fa.select(df, col("k").cast(str).like("99%").alias("m"), ff.length(col("k").cast(str)).alias("n"),
                    engine=e, as_fugue=True).as_arrow()
    assert ST.uploads == before
    assert sum(got.column("m").to_pylist()) == sum(str(i).startswith("99") for i in range(100_000))


def test_twenty_million_rows_ten_million_distinct(e):
    n, m = 20_000_000, 10_000_000
    v = torch.arange(n, dtype=torch.int64, device=DEV) % m * 3 - 7
    codes, _, d = ST.format_values(v, None, pa.int64(), DEV)
    assert len(d) == m
    idx = torch.randint(0, n, (1000,), device=DEV)
    assert [d[c].as_py() for c in codes[idx].tolist()] == [str(x) for x in v[idx].tolist()]
    assert d[0].as_py() == str(-7) and d[m - 1].as_py() == str((m - 1) * 3 - 7)
