"""NTILE, PERCENT_RANK, CUME_DIST, FIRST_VALUE, LAST_VALUE and NTH_VALUE on the H100 (DESIGN §4, §7p): against SQLite
(>= 3.30 for NULLS LAST) row by row in input order, the ColumnMap route against the select route, the value heads at
every column type against the plain-Python reference, edge and large sizes (3 M rows, one 10^6-row peer group, one
10^7-row partition) against numpy, a spy showing the two kernels ran, and bit-identical reruns."""
import sqlite3
from typing import Any, List

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 30), reason="needs SQLite >= 3.30")]
torch = pytest.importorskip("torch")

import test_sql_window_types_gpu as WT  # noqa: E402
from _window_value_oracle import evaluate, ntile_bucket  # noqa: E402
from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import colmap  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402

DEV = torch.device("cuda", 0)
_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


def _device(tbl: pa.Table, items: str, rest: str = "") -> pa.Table:
    return fa.raw_sql(f"SELECT {items} FROM", _df(tbl), rest, engine=_engine(), as_fugue=True).as_arrow()


def _table(rng, n: int, nkeys: int = 5) -> pa.Table:
    """Partition keys with NULLs, an int64 order key t and a float64 one tf (NULLs, NaN, -0.0, ties), int64 and dyadic
    float64 values with NULLs, and vt / vtf, functions of t / tf: peers hold equal values, so a value head under a
    RANGE frame does not depend on how SQLite orders ties."""
    t = rng.integers(0, max(1, n // 4), n)
    tmask = rng.random(n) < 0.05
    tf = rng.integers(-20, 20, n) / 2.0
    tf[rng.random(n) < 0.05] = -0.0
    tf[rng.random(n) < 0.03] = np.nan
    tfmask = rng.random(n) < 0.03
    tf_null = tfmask | np.isnan(tf)
    return pa.table({
        "rid": np.arange(n, dtype=np.int64),
        "ki": pa.array(rng.integers(0, nkeys, n), mask=rng.random(n) < 0.1, type=pa.int64()),
        "ks": pa.array(np.array(["a", "bb", "", "ccc", "d"])[rng.integers(0, 5, n)], mask=rng.random(n) < 0.1),
        "t": pa.array(t, mask=tmask, type=pa.int64()),
        "tf": pa.array(tf, mask=tfmask, type=pa.float64()),
        "vi": pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.15, type=pa.int64()),
        "vf": pa.array(rng.integers(-2**20, 2**20, n) / 4.0, mask=rng.random(n) < 0.15, type=pa.float64()),
        "vt": pa.array(t * 3 - 7, mask=tmask | (t % 5 == 0), type=pa.int64()),
        "vtf": pa.array(np.where(tf_null, 0.0, tf * 2 + 0.25), mask=tf_null | (tf == 1.5), type=pa.float64()),
    })


def _sqlite(tbl: pa.Table, sql: str) -> List[tuple]:
    con = sqlite3.connect(":memory:")
    names = tbl.column_names
    con.execute(f"CREATE TABLE t ({', '.join(names)})")
    rows = [[None if isinstance(x, float) and x != x else x for x in r]
            for r in zip(*[tbl[c].to_pylist() for c in names])]
    con.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})", rows)
    return con.execute(sql).fetchall()


def _rows(res: pa.Table) -> List[tuple]:
    return list(zip(*[res[c].to_pylist() for c in res.column_names]))


def _same_rows(got: List[tuple], want: List[tuple]) -> None:
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for a, b in zip(g, w):  # floats too: PERCENT_RANK and CUME_DIST must equal SQLite's bit for bit
            assert a == b and (a is None) == (b is None) and type(a) is type(b), (g, w)


# (device text, SQLite text): rid is the last SQLite ORDER BY key wherever ties would make its answer arbitrary;
# PERCENT_RANK / CUME_DIST and RANGE frames keep the peers, and the RANGE value heads read vt / vtf
CASES = [
    ("NTILE(4) OVER (PARTITION BY ki ORDER BY t)", "NTILE(4) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid)"),
    ("NTILE(10) OVER (PARTITION BY ks ORDER BY tf DESC)", "NTILE(10) OVER (PARTITION BY ks ORDER BY tf DESC NULLS LAST, rid)"),
    ("NTILE(3000) OVER (PARTITION BY ki ORDER BY t)", "NTILE(3000) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid)"),
    ("NTILE(7) OVER (PARTITION BY ki)", "NTILE(7) OVER (PARTITION BY ki ORDER BY rid)"),
    ("PERCENT_RANK() OVER (PARTITION BY ki ORDER BY t)", "PERCENT_RANK() OVER (PARTITION BY ki ORDER BY t NULLS LAST)"),
    ("PERCENT_RANK() OVER (PARTITION BY ks ORDER BY tf DESC)", "PERCENT_RANK() OVER (PARTITION BY ks ORDER BY tf DESC NULLS LAST)"),
    ("PERCENT_RANK() OVER (ORDER BY t)", "PERCENT_RANK() OVER (ORDER BY t NULLS LAST)"),
    ("PERCENT_RANK() OVER (PARTITION BY ki)", None),
    ("CUME_DIST() OVER (PARTITION BY ki ORDER BY t DESC)", "CUME_DIST() OVER (PARTITION BY ki ORDER BY t DESC NULLS LAST)"),
    ("CUME_DIST() OVER (PARTITION BY ks ORDER BY tf)", "CUME_DIST() OVER (PARTITION BY ks ORDER BY tf NULLS LAST)"),
    ("CUME_DIST() OVER ()", None),
    ("FIRST_VALUE(vi) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING)",
     "FIRST_VALUE(vi) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING)"),
    ("LAST_VALUE(vf) OVER (PARTITION BY ks ORDER BY t DESC ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)",
     "LAST_VALUE(vf) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST, rid ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)"),
    ("NTH_VALUE(vi, 2) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN 1 FOLLOWING AND 1200 FOLLOWING)",
     "NTH_VALUE(vi, 2) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN 1 FOLLOWING AND 1200 FOLLOWING)"),
    ("NTH_VALUE(vf, 3) OVER (PARTITION BY ki ORDER BY t ROWS UNBOUNDED PRECEDING)",
     "NTH_VALUE(vf, 3) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS UNBOUNDED PRECEDING)"),
    ("LAST_VALUE(vi) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN 3 PRECEDING AND UNBOUNDED FOLLOWING)",
     "LAST_VALUE(vi) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN 3 PRECEDING AND UNBOUNDED FOLLOWING)"),
    ("FIRST_VALUE(ks) OVER (PARTITION BY ki ORDER BY t ROWS BETWEEN 1 PRECEDING AND 1 FOLLOWING)",
     "FIRST_VALUE(ks) OVER (PARTITION BY ki ORDER BY t NULLS LAST, rid ROWS BETWEEN 1 PRECEDING AND 1 FOLLOWING)"),
    ("FIRST_VALUE(vi) OVER (PARTITION BY ki)", "FIRST_VALUE(vi) OVER (PARTITION BY ki ORDER BY rid ROWS BETWEEN "
                                               "UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING)"),
    # the default frame with ORDER BY: RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW (LAST_VALUE: the last peer)
    ("LAST_VALUE(vt) OVER (PARTITION BY ki ORDER BY t)", "LAST_VALUE(vt) OVER (PARTITION BY ki ORDER BY t NULLS LAST)"),
    ("FIRST_VALUE(vt) OVER (PARTITION BY ks ORDER BY t DESC)", "FIRST_VALUE(vt) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST)"),
    ("NTH_VALUE(vtf, 2) OVER (PARTITION BY ki ORDER BY tf)", "NTH_VALUE(vtf, 2) OVER (PARTITION BY ki ORDER BY tf NULLS LAST)"),
    ("LAST_VALUE(vt) OVER (PARTITION BY ki ORDER BY t RANGE BETWEEN 5 PRECEDING AND 3 FOLLOWING)",
     "LAST_VALUE(vt) OVER (PARTITION BY ki ORDER BY t NULLS LAST RANGE BETWEEN 5 PRECEDING AND 3 FOLLOWING)"),
    ("FIRST_VALUE(vt) OVER (PARTITION BY ks ORDER BY t DESC RANGE BETWEEN 2 PRECEDING AND CURRENT ROW)",
     "FIRST_VALUE(vt) OVER (PARTITION BY ks ORDER BY t DESC NULLS LAST RANGE BETWEEN 2 PRECEDING AND CURRENT ROW)"),
    ("NTH_VALUE(vtf, 2) OVER (PARTITION BY ki ORDER BY tf RANGE BETWEEN 1.5 PRECEDING AND 2.5 FOLLOWING)",
     "NTH_VALUE(vtf, 2) OVER (PARTITION BY ki ORDER BY tf NULLS LAST RANGE BETWEEN 1.5 PRECEDING AND 2.5 FOLLOWING)"),
    ("NTH_VALUE(vt, 3) OVER (ORDER BY t RANGE BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING)",
     "NTH_VALUE(vt, 3) OVER (ORDER BY t NULLS LAST RANGE BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING)"),
]


def _oracle_select(tbl: pa.Table, cases) -> None:
    dev = ", ".join(f"{d} AS w{i}" for i, (d, _) in enumerate(cases))
    ref = ", ".join(f"{s or d} AS w{i}" for i, (d, s) in enumerate(cases))
    got = _device(tbl, "rid, " + dev)
    assert got["rid"].to_pylist() == list(range(tbl.num_rows))
    _same_rows(_rows(got), _sqlite(tbl, f"SELECT rid, {ref} FROM t ORDER BY rid"))


def test_every_head_matches_sqlite():
    _oracle_select(_table(np.random.default_rng(1), 6000), CASES)


@pytest.mark.parametrize("n", [0, 1, 2, 2047, 2049, 4095, 4097, 6143, 6145])
def test_edge_sizes_match_sqlite(n):
    _oracle_select(_table(np.random.default_rng(n), n, nkeys=2), CASES)


def test_interval_offsets_match_sqlite():
    rng = np.random.default_rng(2)
    n = 3000
    days = rng.integers(0, 400, n)
    d = pa.array(days.astype("datetime64[D]"), mask=rng.random(n) < 0.05)
    tbl = pa.table({"rid": np.arange(n), "k": rng.integers(0, 4, n), "d": d,
                    "v": pa.array(days * 2 + 1, mask=(days % 7 == 0) | pc.is_null(d).to_numpy(zero_copy_only=False))})
    got = _device(tbl, "rid, NTH_VALUE(v, 2) OVER (PARTITION BY k ORDER BY d RANGE BETWEEN INTERVAL '7' DAY PRECEDING "
                       "AND CURRENT ROW) AS a, LAST_VALUE(v) OVER (PARTITION BY k ORDER BY d DESC RANGE BETWEEN "
                       "INTERVAL '3' DAY PRECEDING AND INTERVAL '2' DAY FOLLOWING) AS b")
    dnull = pc.is_null(d).to_numpy(zero_copy_only=False)
    sq = tbl.set_column(2, "d", pa.array([None if m else int(x) for x, m in zip(days, dnull)], pa.int64()))
    want = _sqlite(sq, "SELECT rid, NTH_VALUE(v, 2) OVER (PARTITION BY k ORDER BY d NULLS LAST RANGE BETWEEN 7 "
                       "PRECEDING AND CURRENT ROW), LAST_VALUE(v) OVER (PARTITION BY k ORDER BY d DESC NULLS LAST "
                       "RANGE BETWEEN 3 PRECEDING AND 2 FOLLOWING) FROM t ORDER BY rid")
    _same_rows(_rows(got), want)


def test_several_specs_and_qualify_match_sqlite():
    tbl = _table(np.random.default_rng(3), 8000, nkeys=30)
    got = _device(tbl, "rid, ki, t", "QUALIFY NTILE(10) OVER (PARTITION BY ki ORDER BY t DESC) = 1")
    want = _sqlite(tbl, "SELECT rid, ki, t FROM (SELECT rid, ki, t, NTILE(10) OVER (PARTITION BY ki ORDER BY t DESC "
                        "NULLS LAST, rid) AS q FROM t) WHERE q = 1 ORDER BY rid")
    _same_rows(_rows(got), want)
    got = _device(tbl, "rid, CUME_DIST() OVER (PARTITION BY ks ORDER BY tf) AS c",
                  "QUALIFY c <= 0.5 AND PERCENT_RANK() OVER (PARTITION BY ki ORDER BY t) > 0")
    want = _sqlite(tbl, "SELECT rid, c FROM (SELECT rid, CUME_DIST() OVER (PARTITION BY ks ORDER BY tf NULLS LAST) AS "
                        "c, PERCENT_RANK() OVER (PARTITION BY ki ORDER BY t NULLS LAST) AS p FROM t) WHERE c <= 0.5 AND "
                        "p > 0 ORDER BY rid")
    _same_rows(_rows(got), want)


def test_column_map_route_equals_the_select_route():
    rng = np.random.default_rng(8)
    n = 20_000
    tbl = pa.table({"rid": np.arange(n), "k": pa.array(rng.integers(0, 7, n), mask=rng.random(n) < 0.05),
                    "t": pa.array(rng.integers(0, 3000, n), mask=rng.random(n) < 0.05),
                    "v": pa.array(rng.normal(0, 5.0, n), mask=rng.random(n) < 0.1),
                    "i": pa.array(rng.integers(-100, 100, n), mask=rng.random(n) < 0.1)})
    both = {
        "nt": ("NTILE(10) OVER (PARTITION BY k ORDER BY t)", f.ntile(10)),
        "pr": ("PERCENT_RANK() OVER (PARTITION BY k ORDER BY t)", f.percent_rank()),
        "cd": ("CUME_DIST() OVER (PARTITION BY k ORDER BY t)", f.cume_dist()),
        "lv": ("LAST_VALUE(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)",
               f.last_value(col("v")).over(rows=(-6, 0))),
        "nv": ("NTH_VALUE(i, 2) OVER (PARTITION BY k ORDER BY t RANGE BETWEEN 5 PRECEDING AND 5 FOLLOWING)",
               f.nth_value(col("i"), 2).over(range=(-5, 5))),
        "fv": ("FIRST_VALUE(i) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED "
               "FOLLOWING)", f.first_value(col("i"))),
        "pl": ("LAST_VALUE(i) OVER (PARTITION BY k ORDER BY t)", f.last_value(col("i")).over(range=(None, 0))),
        "rn": ("FIRST_VALUE(v) OVER (PARTITION BY k ORDER BY t ROWS UNBOUNDED PRECEDING)",
               f.first_value(col("v")).over(running=True)),
    }
    sql = _device(tbl, "rid, " + ", ".join(f"{s} AS {nm}" for nm, (s, _) in both.items()))
    schema = "rid:long," + ",".join(f"{nm}:{'double' if pa.types.is_floating(sql.schema.field(nm).type) else 'long'}"
                                    for nm in both)
    cm = fa.transform(_df(tbl), ColumnMap("rid", *[e.alias(nm) for nm, (_, e) in both.items()]), schema=schema,
                      partition=PartitionSpec(by=["k"], presort="t"), engine=_engine(), as_fugue=True).as_arrow()
    cm = cm.take(pc.sort_indices(cm["rid"]))
    for nm in both:
        assert sql[nm].to_pylist() == cm[nm].to_pylist(), nm


def _bits(a: Any) -> list:
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    tp = a.type
    if pa.types.is_floating(tp):
        a = a.view({16: pa.uint16(), 32: pa.uint32(), 64: pa.uint64()}[tp.bit_width])
    elif pa.types.is_temporal(tp):
        a = a.view(pa.int32() if tp.bit_width == 32 else pa.int64())
    return a.to_pylist()


@pytest.mark.parametrize("nm", list(WT.TYPES))
def test_value_heads_at_every_type_match_the_reference(nm):
    tbl = WT._table(3000, seed=5)
    forms = {  # name: (SQL, reference head, n, frame); NULLs sit at frame edges often (10 % NULL values)
        "a": (f"FIRST_VALUE({nm}) OVER (PARTITION BY k ORDER BY o ROWS BETWEEN 2 PRECEDING AND 1 FOLLOWING)",
              "FIRST_VALUE", None, ("rows", -2, 1), True),
        "b": (f"LAST_VALUE({nm}) OVER (PARTITION BY k ORDER BY o DESC RANGE BETWEEN 3 PRECEDING AND CURRENT ROW)",
              "LAST_VALUE", None, ("range", -3, 0), False),
        "c": (f"NTH_VALUE({nm}, 2) OVER (PARTITION BY k)", "NTH_VALUE", 2, ("whole",), True),
        "d": (f"NTH_VALUE({nm}, 4) OVER (PARTITION BY k ORDER BY o)", "NTH_VALUE", 4, ("range", None, 0), True),
        "e": (f"LAST_VALUE({nm}) OVER (ORDER BY o ROWS BETWEEN 3 FOLLOWING AND 5 FOLLOWING)", "LAST_VALUE", None,
              ("rows", 3, 5), True),
    }
    got = _device(tbl, ", ".join(f"{s} AS {k}" for k, (s, *_) in forms.items()))
    parts = tbl["k"].to_pylist()
    keys = tbl["o"].to_pylist()
    rid = list(range(tbl.num_rows))
    for k, (_, head, n, frame, asc) in forms.items():
        pick = evaluate(head, parts if k != "e" else [0] * len(rid), None if frame == ("whole",) else keys, rid,
                        n=n, frame=frame, asc=asc)
        want = tbl[nm].take(pa.array(pick, pa.int64()))
        assert got[k].type == tbl[nm].type, k
        assert _bits(got[k]) == _bits(want), (nm, k)


def test_three_million_rows_match_numpy():
    rng = np.random.default_rng(7)
    n = 3_000_000
    k = rng.integers(0, 1000, n)
    t = rng.integers(0, 1 << 12, n)
    v = rng.integers(-1000, 1000, n)
    tbl = pa.table({"rid": np.arange(n), "k": k, "t": t, "v": v})
    got = _device(tbl, "rid, NTILE(10) OVER (PARTITION BY k ORDER BY t) AS nt, PERCENT_RANK() OVER (PARTITION BY k "
                       "ORDER BY t) AS pr, CUME_DIST() OVER (PARTITION BY k ORDER BY t) AS cd, FIRST_VALUE(v) OVER "
                       "(PARTITION BY k ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) AS fv, NTH_VALUE(v, 2) "
                       "OVER (PARTITION BY k) AS nv")
    order = np.lexsort((np.arange(n), t, k))
    ks, ts, vs = k[order], t[order], v[order]
    start = np.concatenate([[True], ks[1:] != ks[:-1]])
    seg_first = np.maximum.accumulate(np.where(start, np.arange(n), 0))
    seg_end = np.concatenate([np.flatnonzero(start)[1:], [n]])[np.cumsum(start) - 1]
    rows = seg_end - seg_first
    head = start | np.concatenate([[True], ts[1:] != ts[:-1]])
    pf = np.maximum.accumulate(np.where(head, np.arange(n), 0))
    nxt = np.minimum.accumulate(np.where(np.concatenate([head[1:], [True]]), np.arange(n), n)[::-1])[::-1]
    pr = np.where(rows > 1, (pf - seg_first) / np.maximum(rows - 1, 1), 0.0)
    cd = (nxt - seg_first + 1) / rows
    r = np.arange(n) - seg_first
    size = rows // 10
    large = rows - 10 * size
    small = large * (size + 1)
    with np.errstate(divide="ignore"):
        nt = np.where(size == 0, r + 1, np.where(r < small, 1 + r // (size + 1),
                                                 1 + large + (r - small) // np.maximum(size, 1)))
    fv = vs[np.maximum(seg_first, np.arange(n) - 6)]
    inv = np.empty(n, np.int64)
    inv[order] = np.arange(n)
    for c, w in {"nt": nt, "pr": pr, "cd": cd, "fv": fv}.items():
        assert np.array_equal(got[c].to_numpy(zero_copy_only=False), w[inv]), c
    # without ORDER BY a partition keeps input order: its second input row (every partition has >= 2 rows here)
    by_k = np.lexsort((np.arange(n), k))
    inv_k = np.empty(n, np.int64)
    inv_k[by_k] = np.arange(n)
    assert np.array_equal(got["nv"].to_numpy(), v[by_k][seg_first + 1][inv_k])


def test_one_large_peer_group_and_one_large_partition():
    n, g0, g = 10_000_000, 3_000_000, 1_000_000
    t = np.arange(n, dtype=np.int64)
    t[g0:g0 + g] = g0  # one peer group of 10^6 rows, across ~490 tiles
    v = (np.arange(n, dtype=np.int64) * 7) % 1001
    tbl = pa.table({"t": t, "v": v})
    got = _device(tbl, "PERCENT_RANK() OVER (ORDER BY t) AS pr, CUME_DIST() OVER (ORDER BY t) AS cd, "
                       "NTILE(10) OVER (ORDER BY t) AS nt, LAST_VALUE(v) OVER (ORDER BY t) AS lv, "
                       "NTH_VALUE(v, 5) OVER (ORDER BY t RANGE BETWEEN CURRENT ROW AND 2 FOLLOWING) AS nv")
    i = np.arange(n)
    pf = np.where((i >= g0) & (i < g0 + g), g0, i)
    pl = np.where((i >= g0) & (i < g0 + g), g0 + g - 1, i)
    assert np.array_equal(got["pr"].to_numpy(), pf / (n - 1))
    assert np.array_equal(got["cd"].to_numpy(), (pl + 1) / n)
    assert np.array_equal(got["nt"].to_numpy(), i // (n // 10) + 1)
    assert np.array_equal(got["lv"].to_numpy(), v[pl])
    # RANGE [t, t + 2]: from the first peer to the last row with key <= t + 2
    keys = t
    hi = np.searchsorted(keys, keys + 2, side="right") - 1
    j = pf + 4
    nv = got["nv"]
    ok = j <= hi
    assert nv.null_count == int(np.sum(~ok))
    assert np.array_equal(nv.to_numpy(zero_copy_only=False)[ok], v[j[ok]])


def test_kernels_ran_and_nothing_fell_back(monkeypatch):
    calls = {"value": 0, "dist": 0, "gather": 0}
    real_v, real_d, real_g = K.window_value, K.window_distribution, K.gather_rows

    def spy(name, fn):
        def run(*a, **kw):
            calls[name] += 1
            return fn(*a, **kw)
        return run

    inside = []

    def gather(*a, **kw):  # row gathers made while the windows are evaluated
        calls["gather"] += len(inside)
        return real_g(*a, **kw)

    def windows(*a, **kw):
        inside.append(1)
        try:
            return real_w(*a, **kw)
        finally:
            inside.pop()

    real_w = colmap._with_windows
    monkeypatch.setattr(K, "window_value", spy("value", real_v))
    monkeypatch.setattr(K, "window_distribution", spy("dist", real_d))
    monkeypatch.setattr(K, "gather_rows", gather)
    monkeypatch.setattr(colmap, "_with_windows", windows)
    tbl = _table(np.random.default_rng(9), 5000)
    cm = ColumnMap("rid", f.first_value(col("vi")).over(rows=(-2, 2)).alias("a"),
                   f.last_value(col("vf")).over(rows=(-2, 2)).alias("b"), f.nth_value(col("vi"), 3).over(rows=(-2, 2)).alias("c"),
                   f.ntile(4).alias("d"), f.ntile(9).alias("e"), f.percent_rank().alias("p"), f.cume_dist().alias("q"))
    fa.transform(_df(tbl), cm, schema="rid:long,a:long,b:double,c:long,d:long,e:long,p:double,q:double",
                 partition=PartitionSpec(by=["ki"], presort="t"), engine=_engine(), as_fugue=True).as_arrow()
    # one launch for the three value heads of one frame, one for the four distribution heads, no row gather
    assert calls["value"] == 1 and calls["dist"] == 1
    assert calls["gather"] == 0


def test_reruns_are_bit_identical():
    tbl = _table(np.random.default_rng(10), 50_000, nkeys=40)
    items = ", ".join(d + f" AS w{i}" for i, (d, _) in enumerate(CASES))
    a, b = _device(tbl, items), _device(tbl, items)
    for c in a.column_names:
        assert _bits(a[c]) == _bits(b[c]), c


def test_ntile_reference_formula_matches_the_kernel_at_n_past_the_rows():
    offsets = torch.tensor([0, 3, 3, 13], dtype=torch.int64, device=DEV)
    heads = torch.zeros(13, dtype=torch.uint8, device=DEV)
    _, _, nts = K.window_distribution(offsets, heads, False, False, [1, 4, 10, 1 << 63])
    r = [0, 1, 2] + list(range(10))
    rows = [3, 3, 3] + [10] * 10
    for nt, m in zip(nts, [1, 4, 10, 1 << 63]):
        assert nt.tolist() == [ntile_bucket(a, b, m) for a, b in zip(r, rows)]
