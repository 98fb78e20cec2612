"""Window functions in SQL and in ``select / assign / filter`` on the H100 (DESIGN §7p): against SQLite (the
standard library's, >= 3.30 for NULLS LAST) row by row in input order, against the ``ColumnMap`` route of
``fa.transform`` for every window head, the builder API against the same SQL text, edge sizes around a tile
(2048 rows) and a carry chunk, and the ``fb_scatter_rows`` kernel against numpy."""
import math
import sqlite3
from typing import Any, List

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 30), reason="needs SQLite >= 3.30")]
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import all_cols, col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table

DEV = torch.device("cuda", 0)
_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


def _table(rng, n: int, nkeys: int = 5, null_keys: bool = False) -> pa.Table:
    """int64 and string partition keys with NULLs, an int64 order key with ties and NULLs, int64 values and dyadic
    float64 values (multiples of 1/4 below 2^20, so every sum is exact) with NULLs."""
    ki = rng.integers(0, nkeys, n)
    kmask = np.ones(n, bool) if null_keys else rng.random(n) < 0.1
    ks = np.array(["a", "bb", "", "ccc", "d"])[rng.integers(0, 5, n)]
    return pa.table({
        "rid": np.arange(n, dtype=np.int64),
        "ki": pa.array(ki, mask=kmask, type=pa.int64()),
        "ks": pa.array(ks, mask=rng.random(n) < 0.1, type=pa.string()),
        "t": pa.array(rng.integers(0, max(1, n // 4), n), mask=rng.random(n) < 0.05, type=pa.int64()),
        "vi": pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.1, type=pa.int64()),
        "vf": pa.array(rng.integers(-2**20, 2**20, n) / 4.0, mask=rng.random(n) < 0.1, type=pa.float64()),
    })


def _sqlite(tbl: pa.Table, sql: str) -> List[tuple]:
    con = sqlite3.connect(":memory:")
    names = tbl.column_names
    con.execute(f"CREATE TABLE t ({', '.join(names)})")
    con.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})",
                    list(zip(*[tbl[c].to_pylist() for c in names])))
    return con.execute(sql).fetchall()


def _device(tbl: pa.Table, items: str, rest: str = "") -> pa.Table:
    return fa.raw_sql(f"SELECT {items} FROM", _df(tbl), rest, engine=_engine(), as_fugue=True).as_arrow()


def _rows(res: pa.Table) -> List[tuple]:
    return list(zip(*[res[c].to_pylist() for c in res.column_names]))


def _same_rows(got: List[tuple], want: List[tuple]) -> None:
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert len(g) == len(w)
        for a, b in zip(g, w):
            if isinstance(a, float) and isinstance(b, float) and math.isnan(a) and math.isnan(b):
                continue
            assert a == b and (a is None) == (b is None), (g, w)


# (device text, SQLite text): SQLite gets NULLS LAST, and rid as the last ORDER BY key wherever ties would make its
# answer arbitrary; the device breaks ties by input order, which is rid order here
CASES = [
    ("ROW_NUMBER() OVER (PARTITION BY ki ORDER BY t DESC)", "ROW_NUMBER() OVER (PARTITION BY ki ORDER BY t DESC NULLS LAST, rid)"),
    ("RANK() OVER (PARTITION BY ks ORDER BY t)", "RANK() OVER (PARTITION BY ks ORDER BY t NULLS LAST)"),
    ("DENSE_RANK() OVER (PARTITION BY ki ORDER BY t DESC)", "DENSE_RANK() OVER (PARTITION BY ki ORDER BY t DESC NULLS LAST)"),
    ("LAG(vi) OVER (PARTITION BY ki ORDER BY t)", "LAG(vi) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid)"),
    ("LEAD(vf, 2, 0.5) OVER (PARTITION BY ks ORDER BY t DESC)", "LEAD(vf, 2, 0.5) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST, rid)"),
    ("LAG(vi, 3, -1) OVER (ORDER BY t)", "LAG(vi, 3, -1) OVER (ORDER BY t NULLS LAST, rid)"),
    ("SUM(vi) OVER (PARTITION BY ki)", None),
    ("COUNT(vf) OVER (PARTITION BY ks)", None),
    ("COUNT(*) OVER (PARTITION BY ki)", None),
    ("AVG(vf) OVER (PARTITION BY ki)", None),
    ("MIN(vi) OVER (PARTITION BY ks)", None),
    ("MAX(vf) OVER (PARTITION BY ks, ki)", None),
    ("SUM(vf) OVER (PARTITION BY ki ORDER BY t)", "SUM(vf) OVER (PARTITION BY ki ORDER BY t NULLS LAST)"),
    ("COUNT(*) OVER (PARTITION BY ks ORDER BY t DESC)", "COUNT(*) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST)"),
    ("SUM(vi) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)",
     "SUM(vi) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)"),
    ("AVG(vi) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)",
     "AVG(vi) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)"),
    # frames wider than 1024 rows take the frame kernel's other path; SQLite 3.45's MIN / MAX over such sliding frames
    # is not reliable (it disagrees with a direct evaluation), so these use SUM and COUNT
    ("SUM(vi) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN 1500 PRECEDING AND 200 FOLLOWING)",
     "SUM(vi) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN 1500 PRECEDING AND 200 FOLLOWING)"),
    ("COUNT(vf) OVER (ORDER BY t ROWS BETWEEN 3 FOLLOWING AND 1100 FOLLOWING)",
     "COUNT(vf) OVER (ORDER BY t NULLS LAST, rid ROWS BETWEEN 3 FOLLOWING AND 1100 FOLLOWING)"),
    ("SUM(vf) OVER (PARTITION BY ks ORDER BY t DESC ROWS 2 PRECEDING)",
     "SUM(vf) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST, rid ROWS 2 PRECEDING)"),
    ("SUM(vf) OVER (PARTITION BY ki ORDER BY t RANGE BETWEEN 5 PRECEDING AND 3 FOLLOWING)",
     "SUM(vf) OVER (PARTITION BY ki ORDER BY t NULLS LAST RANGE BETWEEN 5 PRECEDING AND 3 FOLLOWING)"),
    ("COUNT(vi) OVER (PARTITION BY ks ORDER BY t DESC RANGE BETWEEN 2 PRECEDING AND CURRENT ROW)",
     "COUNT(vi) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST RANGE BETWEEN 2 PRECEDING AND CURRENT ROW)"),
    ("SUM(vi) OVER ()", None),
    ("vi * 2 - SUM(vi) OVER (PARTITION BY ki % 3)", None),
    ("MIN(vi) OVER (PARTITION BY ki + 1 ORDER BY t * 2 ROWS BETWEEN 1 PRECEDING AND 1 FOLLOWING)",
     "MIN(vi) OVER (PARTITION BY ki + 1 ORDER BY t * 2 NULLS LAST, rid ROWS BETWEEN 1 PRECEDING AND 1 FOLLOWING)"),
]


def _oracle_select(tbl: pa.Table, cases) -> None:
    dev = ", ".join(f"{d} AS w{i}" for i, (d, _) in enumerate(cases))
    ref = ", ".join(f"{s or d} AS w{i}" for i, (d, s) in enumerate(cases))
    got = _device(tbl, "rid, " + dev)
    assert got["rid"].to_pylist() == list(range(tbl.num_rows))  # rows keep their input order
    _same_rows(_rows(got), _sqlite(tbl, f"SELECT rid, {ref} FROM t ORDER BY rid"))


@pytest.mark.parametrize("n", [5000])
def test_every_window_form_matches_sqlite(n):
    _oracle_select(_table(np.random.default_rng(1), n), CASES)


@pytest.mark.parametrize("n", [0, 1, 2, 2047, 2048, 2049, 4095, 4097])
def test_edge_sizes_match_sqlite(n):
    _oracle_select(_table(np.random.default_rng(n), n, nkeys=2), CASES)


def test_all_null_keys_match_sqlite():
    _oracle_select(_table(np.random.default_rng(3), 3000, null_keys=True), CASES[:10])


def test_qualify_matches_a_sqlite_sub_query():
    tbl = _table(np.random.default_rng(4), 6000)
    got = _device(tbl, "rid, ki, t", "QUALIFY ROW_NUMBER() OVER (PARTITION BY ki ORDER BY t DESC) = 1")
    want = _sqlite(tbl, "SELECT rid, ki, t FROM (SELECT rid, ki, t, ROW_NUMBER() OVER (PARTITION BY ki ORDER BY t DESC "
                        "NULLS LAST, rid) AS rn FROM t) WHERE rn = 1 ORDER BY rid")
    _same_rows(_rows(got), want)
    # QUALIFY names an output alias; WHERE runs first
    got = _device(tbl, "rid, vi, SUM(vi) OVER (PARTITION BY ks) AS s", "WHERE vi > -500 QUALIFY s > 0 AND vi < s")
    want = _sqlite(tbl, "SELECT rid, vi, s FROM (SELECT rid, vi, SUM(vi) OVER (PARTITION BY ks) AS s FROM t "
                        "WHERE vi > -500) WHERE s > 0 AND vi < s ORDER BY rid")
    _same_rows(_rows(got), want)


def test_windows_over_group_by_results_match_sqlite():
    tbl = _table(np.random.default_rng(5), 8000, nkeys=40)
    items = ("ki, SUM(vi) AS s, RANK() OVER (ORDER BY SUM(vi) DESC) AS r, "
             "SUM(vi) * 1.0 / SUM(SUM(vi)) OVER () AS share, LAG(SUM(vi)) OVER (ORDER BY ki) AS prev, "
             "DENSE_RANK() OVER (PARTITION BY ki % 2 ORDER BY COUNT(*)) AS dr")
    got = sorted(_rows(_device(tbl, items, "GROUP BY ki HAVING COUNT(*) > 150")), key=lambda r: (r[0] is None, r[0]))
    want = _sqlite(tbl, "SELECT ki, SUM(vi) AS s, RANK() OVER (ORDER BY SUM(vi) DESC) AS r, "
                        "SUM(vi) * 1.0 / SUM(SUM(vi)) OVER () AS share, LAG(SUM(vi)) OVER (ORDER BY ki NULLS LAST) "
                        "AS prev, DENSE_RANK() OVER (PARTITION BY ki % 2 ORDER BY COUNT(*)) AS dr FROM t GROUP BY ki "
                        "HAVING COUNT(*) > 150 ORDER BY ki NULLS LAST")
    _same_rows(got, want)
    # the top 3 groups by total
    top = sorted(_rows(_device(tbl, "ki, SUM(vi) AS s", "GROUP BY ki QUALIFY RANK() OVER (ORDER BY SUM(vi) DESC) <= 3")),
                 key=lambda r: (-r[1], r[0] is None, r[0]))
    want = _sqlite(tbl, "SELECT ki, s FROM (SELECT ki, SUM(vi) AS s, RANK() OVER (ORDER BY SUM(vi) DESC) AS r FROM t "
                        "GROUP BY ki) WHERE r <= 3 ORDER BY s DESC, ki NULLS LAST")
    _same_rows(top, want)
    with pytest.raises(ValueError):  # vi is neither a group key nor aggregated
        _device(tbl, "ki, SUM(vi) AS s, SUM(vi) OVER (PARTITION BY ki) AS w", "GROUP BY ki")


def test_builder_api_matches_the_sql_text():
    tbl = _table(np.random.default_rng(6), 5000)
    rn = f.row_number().over(partition_by=["ki"], order_by=[("t", False)])
    mov = f.avg(col("vi")).over(rows=(-6, 0), partition_by=["ki"], order_by=["t"])
    share = col("vf") / f.sum(col("vf")).over(partition_by=[col("ks")])
    sql = _device(tbl, "rid, ROW_NUMBER() OVER (PARTITION BY ki ORDER BY t DESC) AS rn, AVG(vi) OVER (PARTITION BY ki "
                       "ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) AS mov, vf / SUM(vf) OVER (PARTITION BY ks) "
                       "AS share")
    sel = fa.select(_df(tbl), "rid", rn.alias("rn"), mov.alias("mov"), share.alias("share"), engine=_engine(),
                    as_fugue=True).as_arrow()
    _same_rows(_rows(sel), _rows(sql))
    asg = fa.assign(_df(tbl), rn=rn, mov=mov, share=share, engine=_engine(), as_fugue=True).as_arrow()
    assert asg.column_names == tbl.column_names + ["rn", "mov", "share"]
    _same_rows(_rows(asg.select(["rid", "rn", "mov", "share"])), _rows(sql))
    flt = fa.filter(_df(tbl), rn == 1, engine=_engine(), as_fugue=True).as_arrow()
    _same_rows(_rows(flt), _rows(_device(tbl, "*", "QUALIFY ROW_NUMBER() OVER (PARTITION BY ki ORDER BY t DESC) = 1")))
    piece = fa.raw_sql("SELECT rid,", rn.alias("rn"), "FROM", _df(tbl), engine=_engine(), as_fugue=True).as_arrow()
    _same_rows(_rows(piece), _rows(sql.select(["rid", "rn"])))


def test_three_million_rows_match_pandas():
    rng = np.random.default_rng(7)
    n = 3_000_000
    k = rng.integers(0, 1000, n)
    t = rng.integers(0, 1 << 20, n)
    v = rng.integers(-1000, 1000, n)
    tbl = pa.table({"rid": np.arange(n), "k": pa.array(k, mask=rng.random(n) < 0.01), "t": t, "v": v})
    got = _device(tbl, "rid, ROW_NUMBER() OVER (PARTITION BY k ORDER BY t) AS rn, SUM(v) OVER (PARTITION BY k) AS s, "
                       "SUM(v) OVER (PARTITION BY k ORDER BY t ROWS UNBOUNDED PRECEDING) AS r").to_pandas()
    pdf = tbl.to_pandas().sort_values(["k", "t"], kind="stable", na_position="last")
    g = pdf.groupby("k", dropna=False, sort=False)["v"]
    pdf["rn"], pdf["s"], pdf["r"] = g.cumcount() + 1, g.transform("sum"), g.cumsum()
    pdf = pdf.sort_values("rid")
    for c in ("rn", "s", "r"):
        assert np.array_equal(got[c].to_numpy(), pdf[c].to_numpy()), c


def _bounded(a: np.ndarray, b: np.ndarray, rtol: float) -> bool:
    both = np.isnan(a) & np.isnan(b)
    return bool(np.all(both | np.isclose(a, b, rtol=rtol, atol=1e-12)))


def test_same_result_as_the_column_map_route():
    rng = np.random.default_rng(8)
    n = 20_000
    tbl = pa.table({"rid": np.arange(n), "k": pa.array(rng.integers(0, 7, n), mask=rng.random(n) < 0.05),
                    "t": pa.array(rng.integers(0, 3000, n), mask=rng.random(n) < 0.05),
                    "x": pa.array(rng.normal(50.0, 5.0, n), mask=rng.random(n) < 0.1),
                    "y": pa.array(rng.normal(-3.0, 2.0, n), mask=rng.random(n) < 0.1),
                    "i": pa.array(rng.integers(-100, 100, n), mask=rng.random(n) < 0.1)})
    exact = {  # name: (SQL text, ColumnMap node): integer results, MIN / MAX, counts, ranks, offsets, percentiles
        "si": ("SUM(i) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 2 PRECEDING AND 5 FOLLOWING)",
               f.sum(col("i")).over(rows=(-2, 5))),
        "ci": ("COUNT(i) OVER (PARTITION BY k ORDER BY t)", f.count(col("i")).over(range=(None, 0))),
        "mx": ("MAX(x) OVER (PARTITION BY k ORDER BY t RANGE BETWEEN 10 PRECEDING AND 10 FOLLOWING)",
               f.max(col("x")).over(range=(-10, 10))),
        "mn": ("MIN(i) OVER (PARTITION BY k)", f.min(col("i")).over()),
        "rn": ("ROW_NUMBER() OVER (PARTITION BY k ORDER BY t)", f.row_number()),
        "rk": ("RANK() OVER (PARTITION BY k ORDER BY t)", f.rank()),
        "dr": ("DENSE_RANK() OVER (PARTITION BY k ORDER BY t)", f.dense_rank()),
        "lg": ("LAG(x, 2) OVER (PARTITION BY k ORDER BY t)", f.lag(col("x"), 2)),
        "ld": ("LEAD(i, 1, 0) OVER (PARTITION BY k ORDER BY t)", f.lead(col("i"), 1, 0)),
        "pc": ("PERCENTILE_CONT(0.3) WITHIN GROUP (ORDER BY x) OVER (PARTITION BY k)", f.percentile_cont(col("x"), 0.3).over()),
        "pd": ("PERCENTILE_DISC(0.7) WITHIN GROUP (ORDER BY i) OVER (PARTITION BY k)", f.percentile_disc(col("i"), 0.7).over()),
        "rc": ("REGR_COUNT(y, x) OVER (PARTITION BY k)", f.regr_count(col("y"), col("x")).over()),
    }
    run = "ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW"
    bounded = {  # f64 sums and moments: tile boundaries differ between the routes
        "sx": (f"SUM(x) OVER (PARTITION BY k ORDER BY t {run})", f.sum(col("x")).over(running=True)),
        "ax": ("AVG(x) OVER (PARTITION BY k)", f.avg(col("x")).over()),
        "vs": ("VAR_SAMP(x) OVER (PARTITION BY k)", f.var_samp(col("x")).over()),
        "sd": (f"STDDEV_POP(x) OVER (PARTITION BY k ORDER BY t {run})", f.stddev_pop(col("x")).over(running=True)),
        "co": ("CORR(x, y) OVER (PARTITION BY k)", f.corr(col("x"), col("y")).over()),
        "rs": (f"REGR_SLOPE(y, x) OVER (PARTITION BY k ORDER BY t {run})", f.regr_slope(col("y"), col("x")).over(running=True)),
        "sk": ("SKEWNESS(x) OVER (PARTITION BY k)", f.skewness(col("x")).over()),
        "ku": (f"KURTOSIS(y) OVER (PARTITION BY k ORDER BY t {run})", f.kurtosis(col("y")).over(running=True)),
    }
    both = {**exact, **bounded}
    sql = _device(tbl, "rid, " + ", ".join(f"{s} AS {nm}" for nm, (s, _) in both.items()))
    types = {nm: sql.schema.field(nm).type for nm in both}
    schema = "rid:long," + ",".join(f"{nm}:{pa.types.is_floating(tp) and 'double' or 'long'}" for nm, tp in types.items())
    cm = fa.transform(_df(tbl), ColumnMap("rid", *[e.alias(nm) for nm, (_, e) in both.items()]), schema=schema,
                      partition=PartitionSpec(by=["k"], presort="t"), engine=_engine(), as_fugue=True).as_arrow()
    cm = cm.take(pc.sort_indices(cm["rid"]))
    assert sql["rid"].to_pylist() == list(range(n))
    for nm in exact:
        assert sql[nm].to_pylist() == cm[nm].to_pylist(), nm
    for nm in bounded:
        a = sql[nm].to_numpy(zero_copy_only=False).astype(float)
        b = cm[nm].to_numpy(zero_copy_only=False).astype(float)
        assert np.array_equal(np.isnan(a), np.isnan(b)) and _bounded(a, b, 1e-9), nm


@pytest.mark.parametrize("n", [0, 1, 10_000_000])
def test_scatter_rows_matches_numpy(n):
    rng = np.random.default_rng(n)
    perm = rng.permutation(n).astype(np.int64)
    cols, valid = [], []
    for dt, with_valid in ((np.uint8, False), (np.int16, True), (np.int32, False), (np.float64, True),
                           (np.int64, False), (np.uint8, True)):
        cols.append(rng.integers(0, 200, n).astype(dt))
        valid.append(rng.integers(0, 2, n).astype(np.uint8) if with_valid else None)
    outs, outv = K.scatter_rows([torch.from_numpy(c).to(DEV) for c in cols],
                                [None if v is None else torch.from_numpy(v).to(DEV) for v in valid],
                                torch.from_numpy(perm).to(DEV))
    for c, v, o, ov in zip(cols, valid, outs, outv):
        want = np.empty_like(c)
        want[perm] = c
        assert np.array_equal(o.cpu().numpy(), want)
        assert (ov is None) == (v is None)
        if v is not None:
            wv = np.empty_like(v)
            wv[perm] = v
            assert np.array_equal(ov.cpu().numpy(), wv)
