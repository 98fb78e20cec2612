"""NTILE, PERCENT_RANK, CUME_DIST, FIRST_VALUE, LAST_VALUE and NTH_VALUE without a GPU: the builders and ``over()``
rules, every rejection, every SQL spelling parsed to its node (default frames included), print -> parse as a fixed
point, numpy models of ``fb_window_value`` / ``fb_window_distribution`` against the plain-Python reference, and that
reference against SQLite on small tables with NULLs, ties, NaN and -0.0 under every frame kind."""
import datetime
import math
import random
import sqlite3

import numpy as np
import pyarrow as pa
import pytest

from fugue_b200.colmap import ColumnMap
from fugue_b200.column import (AGGREGATES, SCALARS, DISTRIBUTIONS, VALUE_HEADS, Kind, col, functions as f,
                               is_explicit, to_sql)
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select

from _window_value_oracle import evaluate, model_distribution, model_value, ntile_bucket


def _item(text: str):
    st = _parse_select(text, "FROM t", "SELECT " + text + " FROM t")
    assert len(st.columns) == 1
    return st.columns[0]


def _same(a, b) -> bool:
    return a.fingerprint() == b.fingerprint()


# ---- builders and over() -------------------------------------------------------------------------------------------
def test_heads_are_window_only():
    for h in DISTRIBUTIONS | VALUE_HEADS:
        assert h not in AGGREGATES and h not in SCALARS


def test_builders_and_types():
    sch = Schema("v:float,s:str,k:long")
    assert f.ntile(4).kind == Kind.WINDOW and f.ntile(4).kwargs == {"n": 4}
    assert f.ntile(4).infer_type(sch) == pa.int64()
    assert f.percent_rank().infer_type(sch) == pa.float64() and f.cume_dist().infer_type(sch) == pa.float64()
    for e in (f.first_value(col("v")), f.last_value("v"), f.nth_value(col("v"), 2)):
        assert e.kind == Kind.WINDOW and e.infer_type(sch) == pa.float32()
        assert e.infer_alias().output_name == "v"
    assert f.last_value(col("s")).infer_type(sch) == pa.string()
    assert f.nth_value("v", 3).kwargs == {"n": 3}
    # a bare node runs over the whole partition in a ColumnMap
    ColumnMap("k", f.first_value(col("v")).alias("a"), f.ntile(3).alias("b"), f.percent_rank().alias("c"),
              f.last_value(col("v")).over(rows=(-6, 0)).alias("d"), f.nth_value(col("v"), 2).over(range=(-3, 0)).alias("e"))


@pytest.mark.parametrize("bad", [0, -1, 2.5, None, True, "2", col("k")])
def test_n_must_be_a_positive_int(bad):
    with pytest.raises(ValueError):
        f.ntile(bad)
    with pytest.raises(ValueError):
        f.nth_value(col("v"), bad)


def test_value_over_takes_every_aggregate_frame():
    v = col("v")
    assert f.last_value(v).over(rows=(-6, 0)).kwargs == {"rows": (-6, 0)}
    assert f.last_value(v).over(rows=(None, 0)).kwargs == {"running": True}
    assert f.last_value(v).over(running=True).kwargs == {"running": True}
    assert f.last_value(v).over(rows=(None, None)).kwargs == {"running": False}
    assert f.first_value(v).over(range=(-1.5, 2)).kwargs == {"range": (-1.5, 2)}
    assert f.first_value(v).over(range=(None, None)).kwargs == {"running": False}
    assert f.first_value(v).over(range=(datetime.timedelta(0), None)).kwargs == {"range": (0, None)}
    e = f.nth_value(v, 2).over(rows=(-2, 2), partition_by=["k"], order_by=[("t", False)])
    assert is_explicit(e) and e.kwargs["n"] == 2 and e.kwargs["rows"] == (-2, 2)
    assert _same(f.first_value(v).over(partition_by=["k"], order_by=["t"]),
                 f.first_value(v).over(running=False, partition_by=["k"], order_by=["t"]))


@pytest.mark.parametrize("make", [
    lambda: f.last_value(col("v")).over(rows=(2, 1)),
    lambda: f.last_value(col("v")).over(rows=(0, 1), running=True),
    lambda: f.last_value(col("v")).over(rows=(0, 1), range=(0, 1)),
    lambda: f.last_value(col("v")).over(running=1),
    lambda: f.last_value(col("v")).over(rows=(0.5, 1)),
    lambda: f.last_value(col("v")).over(range=(float("inf"), None)),
    lambda: f.last_value(col("v")).over(rows=(-1, 0)).over(rows=(-2, 0)),
    lambda: f.last_value(col("v")).over(partition_by=["k"]).over(partition_by=["j"]),
    lambda: f.first_value(col("v")).over(range=(-1, 0), order_by=["t", "u"]),
    lambda: f.ntile(2).over(rows=(-1, 0), order_by=["t"]),
    lambda: f.percent_rank().over(running=True, order_by=["t"]),
    lambda: f.cume_dist().over(range=(None, 0), order_by=["t"]),
    lambda: f.first_value("*"),
    lambda: f.first_value(f.sum(col("v"))),
    lambda: f.first_value(f.row_number().over(order_by=["t"])),
    lambda: f.ntile(2).over(),
])
def test_over_rejections(make):
    with pytest.raises(ValueError):
        make()


# ---- SQL -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("text,node", [
    ("NTILE(4) OVER (PARTITION BY k ORDER BY t) AS q", f.ntile(4).over(partition_by=["k"], order_by=["t"]).alias("q")),
    ("NTILE(10) OVER () AS q", f.ntile(10).over(partition_by=[]).alias("q")),
    ("PERCENT_RANK() OVER (PARTITION BY k ORDER BY t DESC) AS p",
     f.percent_rank().over(partition_by=["k"], order_by=[("t", False)]).alias("p")),
    ("CUME_DIST() OVER (ORDER BY t NULLS LAST) AS c", f.cume_dist().over(order_by=["t"]).alias("c")),
    # the default frame with ORDER BY: RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW
    ("FIRST_VALUE(v) OVER (PARTITION BY k ORDER BY t) AS a",
     f.first_value(col("v")).over(range=(None, 0), partition_by=["k"], order_by=["t"]).alias("a")),
    ("LAST_VALUE(v) OVER (ORDER BY t DESC) AS a", f.last_value(col("v")).over(range=(None, 0), order_by=[("t", False)]).alias("a")),
    # without ORDER BY: the whole partition
    ("LAST_VALUE(v) OVER (PARTITION BY k) AS a", f.last_value(col("v")).over(partition_by=["k"]).alias("a")),
    ("LAST_VALUE(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) AS a",
     f.last_value(col("v")).over(rows=(-6, 0), partition_by=["k"], order_by=["t"]).alias("a")),
    ("FIRST_VALUE(v) OVER (ORDER BY t ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING) AS a",
     f.first_value(col("v")).over(order_by=["t"]).alias("a")),
    ("FIRST_VALUE(v) OVER (ORDER BY t ROWS UNBOUNDED PRECEDING) AS a",
     f.first_value(col("v")).over(running=True, order_by=["t"]).alias("a")),
    ("NTH_VALUE(v, 2) OVER (PARTITION BY k ORDER BY t RANGE BETWEEN 5 PRECEDING AND 2 FOLLOWING) AS a",
     f.nth_value(col("v"), 2).over(range=(-5, 2), partition_by=["k"], order_by=["t"]).alias("a")),
    ("NTH_VALUE(v, 3) FROM FIRST RESPECT NULLS OVER (ORDER BY d RANGE BETWEEN INTERVAL '7' DAY PRECEDING AND CURRENT ROW) AS a",
     f.nth_value(col("v"), 3).over(range=(-datetime.timedelta(days=7), 0), order_by=["d"]).alias("a")),
    ("FIRST_VALUE(v) RESPECT NULLS OVER (ORDER BY t RANGE BETWEEN 0.5 PRECEDING AND 0.5 FOLLOWING) AS a",
     f.first_value(col("v")).over(range=(-0.5, 0.5), order_by=["t"]).alias("a")),
    ("LAST_VALUE(v * 2) OVER (PARTITION BY k % 3) AS a",
     f.last_value(col("v") * 2).over(partition_by=[col("k") % 3]).alias("a")),
])
def test_every_sql_spelling_gives_its_node(text, node):
    got = _item(text)
    assert _same(got, node), (to_sql(got), to_sql(node))


@pytest.mark.parametrize("text,err", [
    ("NTILE(0) OVER (ORDER BY t)", ValueError),
    ("NTILE(-2) OVER (ORDER BY t)", ValueError),
    ("NTILE(1.5) OVER (ORDER BY t)", ValueError),
    ("NTILE(NULL) OVER (ORDER BY t)", ValueError),
    ("NTH_VALUE(v, 0) OVER (ORDER BY t)", ValueError),
    ("NTH_VALUE(v) OVER (ORDER BY t)", ValueError),
    ("NTILE(v) OVER (ORDER BY t)", NotImplementedError),
    ("NTH_VALUE(v, k) OVER (ORDER BY t)", NotImplementedError),
    ("NTH_VALUE(v, 1 + 1) OVER (ORDER BY t)", NotImplementedError),
    ("FIRST_VALUE(v) IGNORE NULLS OVER (ORDER BY t)", NotImplementedError),
    ("LAST_VALUE(v IGNORE NULLS) OVER (ORDER BY t)", NotImplementedError),
    ("NTH_VALUE(v, 2) FROM LAST OVER (ORDER BY t)", NotImplementedError),
    ("NTILE(3)", NotImplementedError),
    ("PERCENT_RANK()", NotImplementedError),
    ("FIRST_VALUE(v)", NotImplementedError),
    ("CUME_DIST() OVER (ORDER BY t ROWS 2 PRECEDING)", ValueError),
    ("NTILE(2) OVER (ORDER BY t RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)", ValueError),
    ("FIRST_VALUE(v) OVER (ORDER BY t GROUPS 2 PRECEDING)", NotImplementedError),
    ("LAST_VALUE(v) OVER (ORDER BY t ROWS 2 PRECEDING EXCLUDE TIES)", NotImplementedError),
    ("FIRST_VALUE(v) OVER (ORDER BY t, u RANGE BETWEEN 1 PRECEDING AND CURRENT ROW)", ValueError),
])
def test_sql_rejections(text, err):
    with pytest.raises(err):
        _item(text)


def _random_node(rng: random.Random):
    spec = {"partition_by": rng.choice([[], ["k"], [col("k") % 3]]),
            "order_by": rng.choice([[], ["t"], [("t", False)], ["t", ("u", False)]])}
    head = rng.choice(sorted(DISTRIBUTIONS | VALUE_HEADS))
    if head in DISTRIBUTIONS:
        node = {"NTILE": lambda: f.ntile(rng.randint(1, 20)), "PERCENT_RANK": f.percent_rank,
                "CUME_DIST": f.cume_dist}[head]()
        return node.over(**spec)
    arg = rng.choice([col("v"), col("v") + 1, col("s")])
    node = {"FIRST_VALUE": lambda: f.first_value(arg), "LAST_VALUE": lambda: f.last_value(arg),
            "NTH_VALUE": lambda: f.nth_value(arg, rng.randint(1, 5))}[head]()
    frames = [{}, {"running": True}, {"rows": (rng.randint(-5, 0), rng.randint(0, 5))}, {"rows": (None, 2)},
              {"rows": (3, None)}, {"range": (None, 0)}, {"range": (0, None)}]
    if len(spec["order_by"]) == 1:
        frames += [{"range": (-rng.randint(1, 9), rng.randint(0, 9))}, {"range": (-2.5, 0)}]
    return node.over(**rng.choice(frames), **spec)


def test_print_parse_fixed_point_on_random_trees():
    rng = random.Random(11)
    for _ in range(400):
        e = _random_node(rng)
        if rng.random() < 0.3:
            e = e * 2 + 1
        e = e.alias("w")
        text = to_sql(e)
        back = _item(text)
        assert _same(back, e), (text, to_sql(back))
        assert to_sql(back) == text


# ---- kernel models against the reference ---------------------------------------------------------------------------
def _sorted_case(rng: np.random.Generator, nparts: int, n: int, distinct: int):
    """Rows already sorted by (partition, key), as the kernels see them."""
    part = np.sort(rng.integers(0, nparts, n))
    key = rng.integers(0, distinct, n)
    order = np.lexsort((key, part))
    part, key = part[order], key[order]
    offsets = np.concatenate([[0], np.flatnonzero(np.diff(part)) + 1, [n]]).astype(np.int64) if n else np.zeros(1, np.int64)
    heads = np.zeros(n, np.uint8)
    if n:
        heads[0] = 1
        heads[1:] = (part[1:] != part[:-1]) | (key[1:] != key[:-1])
    return part, key, offsets, heads


@pytest.mark.parametrize("n,nparts,distinct,tile", [(0, 1, 1, 8), (1, 1, 1, 8), (37, 3, 4, 8), (200, 5, 3, 16),
                                                     (500, 1, 1, 16), (513, 2, 2, 32), (300, 40, 50, 8)])
def test_distribution_model_matches_the_reference(n, nparts, distinct, tile):
    rng = np.random.default_rng(n + nparts)
    part, key, offsets, heads = _sorted_case(rng, nparts, n, distinct)
    # the kernel needs no head at a segment start: drop some of them
    if n:
        heads[offsets[:-1][rng.random(len(offsets) - 1) < 0.5]] = 0
    ntiles = [1, 3, 7, n + 5]
    pr, cd, nts = model_distribution(offsets, heads, ntiles, tile)
    p, k = part.tolist(), key.tolist()
    assert pr.tolist() == evaluate("PERCENT_RANK", p, k)
    assert cd.tolist() == evaluate("CUME_DIST", p, k)
    for nt, m in zip(nts, ntiles):
        assert nt.tolist() == evaluate("NTILE", p, k, n=m)


def test_ntile_buckets_past_the_row_count():
    assert [ntile_bucket(r, 3, 10) for r in range(3)] == [1, 2, 3]
    assert [ntile_bucket(r, 10, 4) for r in range(10)] == [1, 1, 1, 2, 2, 2, 3, 3, 4, 4]
    assert [ntile_bucket(r, 7, 7) for r in range(7)] == list(range(1, 8))
    assert [ntile_bucket(r, 5, (1 << 63) - 1) for r in range(5)] == [1, 2, 3, 4, 5]


@pytest.mark.parametrize("frame", [("whole",), ("running",), ("rows", -3, 0), ("rows", 2, 5), ("rows", -4, -1),
                                   ("rows", None, 1), ("rows", -1, None), ("rows", 0, 0)])
@pytest.mark.parametrize("head,nth", [("FIRST_VALUE", 1), ("LAST_VALUE", 0), ("NTH_VALUE", 2), ("NTH_VALUE", 5),
                                      ("NTH_VALUE", 1 << 62)])
def test_value_model_rows_frames_match_the_reference(frame, head, nth):
    rng = np.random.default_rng(3)
    n = 120
    part, key, offsets, _ = _sorted_case(rng, 6, n, 40)
    vals = rng.integers(-99, 99, n)
    valid = (rng.random(n) > 0.2).astype(np.uint8)
    start, end = {"whole": (None, None), "running": (None, 0)}.get(frame[0], frame[1:])
    got, ok = model_value(offsets, None, None, start, end, vals, valid, nth)
    want = evaluate(head, part.tolist(), key.tolist(), [int(v) if m else None for v, m in zip(vals, valid)],
                    n=nth, frame=frame)
    assert [int(g) if o else None for g, o in zip(got, ok)] == want


@pytest.mark.parametrize("frame", [("range", -3, 0), ("range", None, 0), ("range", 0, None), ("range", 2, 6),
                                   ("range", -5, -2)])
@pytest.mark.parametrize("asc", [True, False])
def test_value_model_bound_frames_match_the_reference(frame, asc):
    rng = np.random.default_rng(4)
    n = 150
    part = np.sort(rng.integers(0, 4, n))
    key = [None if rng.random() < 0.1 else int(x) for x in rng.integers(0, 30, n)]
    vals = rng.integers(-99, 99, n)
    valid = (rng.random(n) > 0.2).astype(np.uint8)
    vlist = [int(v) if m else None for v, m in zip(vals, valid)]
    # lay the rows out in the reference's sorted order and give the kernel each row's [lo, hi]
    from _window_value_oracle import _partitions, frame_bounds, _norm
    order, lo, hi = [], [], []
    for rows in _partitions(part.tolist(), key, asc):
        ks = [_norm(key[i]) for i in rows]
        base = len(order)
        for p in range(len(rows)):
            a, b = frame_bounds(ks, p, frame, asc)
            lo.append(base + a)
            hi.append(base + b)
        order.extend(rows)
    order = np.array(order)
    for head, nth in (("FIRST_VALUE", 1), ("LAST_VALUE", 0), ("NTH_VALUE", 3)):
        got, ok = model_value(np.array([0, n]), np.array(lo), np.array(hi), None, None, vals[order], valid[order], nth)
        want = evaluate(head, part.tolist(), key, vlist, n=nth, frame=frame, asc=asc)
        assert [int(g) if o else None for g, o in zip(got, ok)] == [want[i] for i in order]


# ---- the reference against SQLite ----------------------------------------------------------------------------------
def _table(rng: random.Random, n: int):
    rows = []
    for rid in range(n):
        t = rng.choice([None, float("nan"), -0.0, 0.0, 1.0, 1.5, 2.0, 3.0, 7.0, 7.5, 10.0])
        rows.append({"rid": rid, "k": rng.choice([None, 1, 2, 3]), "t": t,
                     # v is a function of t (NULL for a NULL or NaN t, and sometimes else): peers carry equal values,
                     # so the value heads under RANGE frames do not depend on how SQLite orders ties
                     "v": None if t is None or math.isnan(t) or t == 3.0 else int(t * 4) - 3,
                     "w": rng.choice([None, 5, 6, 7, 8])})
    return rows


def _sqlite(rows, sql: str):
    con = sqlite3.connect(":memory:")
    con.execute("CREATE TABLE x (rid INTEGER, k INTEGER, t REAL, v INTEGER, w INTEGER)")
    con.executemany("INSERT INTO x VALUES (?, ?, ?, ?, ?)",
                    [(r["rid"], r["k"], None if r["t"] is not None and math.isnan(r["t"]) else r["t"], r["v"], r["w"])
                     for r in rows])
    return [x[0] for x in con.execute(f"SELECT {sql} FROM x ORDER BY rid").fetchall()]


_SQLITE_CASES = [
    # (SQLite text, reference arguments): ROWS-like frames and NTILE get rid as the last order key
    ("NTILE(3) OVER (PARTITION BY k ORDER BY t NULLS LAST, rid)", ("NTILE", {"n": 3})),
    ("NTILE(50) OVER (PARTITION BY k ORDER BY t DESC NULLS LAST, rid)", ("NTILE", {"n": 50, "asc": False})),
    ("NTILE(4) OVER (PARTITION BY k ORDER BY rid)", ("NTILE", {"n": 4, "nokey": True})),
    ("PERCENT_RANK() OVER (PARTITION BY k ORDER BY t NULLS LAST)", ("PERCENT_RANK", {})),
    ("PERCENT_RANK() OVER (PARTITION BY k ORDER BY t DESC NULLS LAST)", ("PERCENT_RANK", {"asc": False})),
    ("PERCENT_RANK() OVER (PARTITION BY k)", ("PERCENT_RANK", {"nokey": True})),
    ("CUME_DIST() OVER (PARTITION BY k ORDER BY t NULLS LAST)", ("CUME_DIST", {})),
    ("CUME_DIST() OVER (ORDER BY t DESC NULLS LAST)", ("CUME_DIST", {"asc": False, "onepart": True})),
    ("CUME_DIST() OVER (PARTITION BY k)", ("CUME_DIST", {"nokey": True})),
    ("FIRST_VALUE(w) OVER (PARTITION BY k ORDER BY t NULLS LAST, rid ROWS BETWEEN 2 PRECEDING AND 1 FOLLOWING)",
     ("FIRST_VALUE", {"frame": ("rows", -2, 1), "arg": "w"})),
    ("LAST_VALUE(w) OVER (PARTITION BY k ORDER BY t NULLS LAST, rid ROWS BETWEEN 2 PRECEDING AND 1 FOLLOWING)",
     ("LAST_VALUE", {"frame": ("rows", -2, 1), "arg": "w"})),
    ("NTH_VALUE(w, 2) OVER (PARTITION BY k ORDER BY t DESC NULLS LAST, rid ROWS BETWEEN 1 FOLLOWING AND 4 FOLLOWING)",
     ("NTH_VALUE", {"n": 2, "frame": ("rows", 1, 4), "arg": "w", "asc": False})),
    ("NTH_VALUE(w, 3) OVER (PARTITION BY k ORDER BY t NULLS LAST, rid ROWS UNBOUNDED PRECEDING)",
     ("NTH_VALUE", {"n": 3, "frame": ("running",), "arg": "w"})),
    ("LAST_VALUE(w) OVER (PARTITION BY k ORDER BY t NULLS LAST, rid ROWS BETWEEN UNBOUNDED PRECEDING AND "
     "UNBOUNDED FOLLOWING)", ("LAST_VALUE", {"arg": "w"})),
    ("FIRST_VALUE(v) OVER (PARTITION BY k ORDER BY t NULLS LAST)", ("FIRST_VALUE", {"frame": ("range", None, 0)})),
    ("LAST_VALUE(v) OVER (PARTITION BY k ORDER BY t NULLS LAST)", ("LAST_VALUE", {"frame": ("range", None, 0)})),
    ("LAST_VALUE(v) OVER (PARTITION BY k ORDER BY t DESC NULLS LAST)",
     ("LAST_VALUE", {"frame": ("range", None, 0), "asc": False})),
    ("NTH_VALUE(v, 2) OVER (PARTITION BY k ORDER BY t NULLS LAST RANGE BETWEEN 1.5 PRECEDING AND 2 FOLLOWING)",
     ("NTH_VALUE", {"n": 2, "frame": ("range", -1.5, 2)})),
    ("FIRST_VALUE(v) OVER (PARTITION BY k ORDER BY t DESC NULLS LAST RANGE BETWEEN 1 PRECEDING AND CURRENT ROW)",
     ("FIRST_VALUE", {"frame": ("range", -1, 0), "asc": False})),
    ("LAST_VALUE(v) OVER (ORDER BY t NULLS LAST RANGE BETWEEN CURRENT ROW AND 3 FOLLOWING)",
     ("LAST_VALUE", {"frame": ("range", 0, 3), "onepart": True})),
    ("NTH_VALUE(v, 4) OVER (PARTITION BY k ORDER BY t NULLS LAST RANGE BETWEEN UNBOUNDED PRECEDING AND 0.5 PRECEDING)",
     ("NTH_VALUE", {"n": 4, "frame": ("range", None, -0.5)})),
]


@pytest.mark.parametrize("sql,ref", _SQLITE_CASES, ids=[c[0][:60] for c in _SQLITE_CASES])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reference_matches_sqlite(sql, ref, seed):
    rng = random.Random(seed)
    rows = _table(rng, rng.randint(1, 60))
    head, kw = ref
    parts = [None for _ in rows] if kw.get("onepart") else [r["k"] for r in rows]
    keys = None if kw.get("nokey") else [r["t"] for r in rows]
    vals = [r[kw.get("arg", "v")] for r in rows]
    got = evaluate(head, parts, keys, vals, n=kw.get("n"), frame=kw.get("frame", ("whole",)), asc=kw.get("asc", True))
    want = _sqlite(rows, sql)
    assert got == want, (sql, got, want)
