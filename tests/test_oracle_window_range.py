"""The RANGE-frame reference (tests/_range_oracle.py) on the CPU: its loop against its vectorised form, whole maps
against the standard library's SQLite (RANGE offsets since 3.28, NULLS LAST since 3.30), and ``range=(None, 0)``
against a running aggregate read at each peer group's last row."""
import math
import sqlite3
from collections import OrderedDict

import numpy as np
import pyarrow as pa
import pytest

import _range_oracle as R
from fugue_b200.column import _frame_bound, all_cols, col, functions as f
from oracle import window as W

pytestmark = pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 30), reason="needs SQLite >= 3.30")

OPS = ["COUNT", "SUM_I64", "SUM_F64", "MIN_I64", "MAX_I64", "MIN_F64", "MAX_F64"]


def _sorted_segments(rng, n, cls, ascending):
    """Random segments, each sorted by a random key with ties, NULL keys last."""
    cut = np.sort(rng.integers(0, n + 1, int(rng.integers(0, 6))))
    off = np.concatenate([[0], cut, [n]]).astype(np.int64)
    if cls == "F64":
        k = rng.choice([-np.inf, -3.0, -1.5, -0.0, 0.0, 1.0, 2.5, 7.0, np.inf, 1e308, -1e308, 5e-324], n)
    elif cls == "U64":
        k = rng.choice(np.array([0, 1, 5, 6, 2**63, 2**63 + 2, 2**64 - 1, 2**64 - 3], dtype=np.uint64), n).view(np.int64)
    else:
        k = rng.choice(np.array([-2**63, -2**63 + 2, -5, 0, 3, 4, 7, 2**63 - 1, 2**63 - 2]), n).astype(np.int64)
    ok = rng.random(n) < 0.8
    for s in range(len(off) - 1):
        a, b = off[s], off[s + 1]
        kk = k[a:b].view(np.uint64) if cls == "U64" else k[a:b]
        v, iv = np.flatnonzero(ok[a:b]), np.flatnonzero(~ok[a:b])
        vs = v[np.argsort(kk[v], kind="stable")]
        o = np.concatenate([vs if ascending else vs[::-1], iv]).astype(int)
        k[a:b], ok[a:b] = k[a:b][o], ok[a:b][o]
    return off, k, ok


@pytest.mark.parametrize("cls", ["I64", "U64", "F64"])
@pytest.mark.parametrize("ascending", [True, False])
def test_bounds_loop_matches_vectorised(cls, ascending):
    rng = np.random.default_rng(len(cls) + 7 * ascending + ord(cls[0]))
    frames = [(0, 0), (-1, 1), (1, 3), (-3, -1), (None, 0), (0, None), (None, -2), (2, None),
              (-2**63, 2**63 - 1), (2**63 - 1, 2**63 - 1), (-2**63, -2**63)]
    if cls == "F64":
        frames += [(-0.5, 1e308), (-1e308, -1e308)]
    for _ in range(60):
        off, k, ok = _sorted_segments(rng, int(rng.integers(0, 50)), cls, ascending)
        for s, e in frames:
            a = R.range_bounds(off, k, ok, cls, ascending, s, e, loop=True)
            b = R.range_bounds(off, k, ok, cls, ascending, s, e, loop=False)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (s, e)


def test_bounds_example_at_the_int64_edges():
    off = np.array([0, 3], dtype=np.int64)
    k = np.array([2**63 - 3, 2**63 - 2, 2**63 - 1], dtype=np.int64)
    lo, hi = R.range_bounds(off, k, None, "I64", True, 1, 3)
    assert hi[2] < lo[2]  # no key above INT64_MAX: empty, where a saturating sum would keep the row itself
    assert (lo[0], hi[0]) == (1, 2)
    lo, hi = R.range_bounds(off, k[::-1].copy(), None, "I64", False, -3, -1)  # DESC: k - (-1) .. k - (-3)
    assert hi[0] < lo[0] and (lo[2], hi[2]) == (0, 1)


def test_aggregate_loop_matches_vectorised():
    rng = np.random.default_rng(3)
    for _ in range(40):
        n = int(rng.integers(0, 90))
        lo, hi = rng.integers(-5, n + 5, n), rng.integers(-5, n + 5, n)
        for op in OPS:
            if op.endswith("F64"):
                v = (rng.integers(-2**20, 2**20, n) * 2.0**-10).view(np.int64)
            else:
                v = rng.integers(-2**63, 2**63 - 1, n)
            m = rng.random(n) < 0.7
            a = R.bounded_aggregate(None if op == "COUNT" else v, m, lo, hi, op, loop=True)
            b = R.bounded_aggregate(None if op == "COUNT" else v, m, lo, hi, op, loop=False)
            assert np.array_equal(a[1], b[1]), op
            if op != "COUNT":
                assert np.array_equal(a[0], b[0]), op


# ---- against SQLite ---------------------------------------------------------------------------------
FRAMES = [(-3, 0), (-2, 2), (1, 3), (-3, -1), (0, 0), (None, 0), (0, None), (None, -1), (2, None), (None, 5),
          (-4, None)]


def _table(rng, n, kind):
    key = rng.integers(0, 4, n)
    if kind == "int":
        t = pa.array(rng.integers(-6, 7, n), mask=rng.random(n) < 0.12)
    else:
        t = pa.array(rng.choice([-np.inf, -2.5, -1.0, -0.0, 0.0, 0.5, 1.0, 1.5, 3.0, np.inf], n),
                     mask=rng.random(n) < 0.12)
    v = pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.15)
    x = pa.array(rng.standard_normal(n), mask=rng.random(n) < 0.15)
    return pa.table({"rid": np.arange(n), "key": key, "t": t, "v": v, "x": x})


def _sqlite(tbl, frame, ascending):
    con = sqlite3.connect(":memory:")
    con.execute("CREATE TABLE d (rid INTEGER, key INTEGER, t, v INTEGER, x REAL)")
    con.executemany("INSERT INTO d VALUES (?, ?, ?, ?, ?)", zip(*[tbl.column(c).to_pylist() for c in tbl.column_names]))
    over = f"OVER (PARTITION BY key ORDER BY t {'ASC' if ascending else 'DESC'} NULLS LAST RANGE BETWEEN " \
           f"{_frame_bound(frame[0], 'PRECEDING')} AND {_frame_bound(frame[1], 'FOLLOWING')})"
    q = f"SELECT rid, COUNT(v) {over}, COUNT(*) {over}, SUM(v) {over}, MIN(v) {over}, MAX(v) {over}, " \
        f"MIN(x) {over}, MAX(x) {over}, SUM(x) {over}, AVG(x) {over} FROM d ORDER BY rid"
    rows = con.execute(q).fetchall()
    con.close()
    return list(zip(*rows))


@pytest.mark.parametrize("kind", ["int", "float"])
@pytest.mark.parametrize("ascending", [True, False])
def test_window_map_matches_sqlite(kind, ascending):
    rng = np.random.default_rng(11 + len(kind) + ascending)
    tbl = _table(rng, 300, kind)
    for frame in FRAMES + ([(-0.5, 0.5), (-1.5, -0.5)] if kind == "float" else []):
        cols = [f.count(col("v")).over(range=frame).alias("cv"), f.count(all_cols()).over(range=frame).alias("cs"),
                f.sum(col("v")).over(range=frame).alias("sv"), f.min(col("v")).over(range=frame).alias("mnv"),
                f.max(col("v")).over(range=frame).alias("mxv"), f.min(col("x")).over(range=frame).alias("mnx"),
                f.max(col("x")).over(range=frame).alias("mxx"), f.sum(col("x")).over(range=frame).alias("sx"),
                f.avg(col("x")).over(range=frame).alias("ax")]
        got = R.window_map(tbl, ["key"], OrderedDict(t=ascending), [col("rid")] + cols)
        exp = _sqlite(tbl, frame, ascending)
        assert got["rid"] == list(exp[0])
        for name, e in zip(["cv", "cs", "sv", "mnv", "mxv", "mnx", "mxx"], exp[1:8]):
            assert got[name] == list(e), (frame, name)
        for name, e in zip(["sx", "ax"], exp[8:]):
            for a, b in zip(got[name], e):
                assert (a is None) == (b is None), (frame, name)
                if a is not None:
                    assert math.isclose(a, b, rel_tol=1e-12, abs_tol=1e-12), (frame, name, a, b)


def test_range_to_current_row_is_the_running_value_at_the_last_peer():
    rng = np.random.default_rng(5)
    tbl = _table(rng, 400, "int")
    for ascending in (True, False):
        got = R.window_map(tbl, ["key"], OrderedDict(t=ascending),
                           [col("rid"), col("key"), col("t"), f.sum(col("v")).over(range=(None, 0)).alias("r"),
                            f.sum(col("v")).over(running=True).alias("run")])
        # the running value of the last row of every (key, t) peer group, NULL t a group of its own
        last = {}
        order = W.S.argsort(tbl, OrderedDict(key=True, t=ascending), "last")
        for i in order.tolist():
            last[(got["key"][i], got["t"][i])] = got["run"][i]
        assert got["r"] == [last[(k_, t_)] for k_, t_ in zip(got["key"], got["t"])]
