"""oracle/window.py (the exact statement of the window functions of a ColumnMap) against a naive per-group Python
loop, and against pandas where pandas means the same thing.  CPU only."""
import math
import struct
from collections import OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from fugue_b200.column import all_cols, col, functions as f
from oracle import window as W


def _table(n: int, seed: int, nulls: bool = True) -> pa.Table:
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 6, n)
    p = rng.integers(0, 5, n)                       # presort with ties
    v = rng.integers(-50, 50, n)
    x = np.round(rng.standard_normal(n), 3)
    s = np.array(["a", "b", "c", "d"], dtype=object)[rng.integers(0, 4, n)]
    m = lambda q: (rng.random(n) < q) if nulls else np.zeros(n, dtype=bool)  # noqa: E731
    return pa.table({"rid": pa.array(np.arange(n)), "k": pa.array(k, mask=m(0.1)), "p": pa.array(p, mask=m(0.1)),
                     "v": pa.array(v, mask=m(0.2)), "x": pa.array(x, mask=m(0.2)),
                     "s": pa.array(list(s), mask=m(0.2), type=pa.string())})


def _naive(t: pa.Table, keys, presort, fn):
    """Group rows by key tuple in Python, sort each group by presort (NULLs last, stable), call ``fn(rows)`` with
    the group's rows (dicts) in order; ``fn`` returns one value per row.  Result keyed by ``rid``."""
    rows = t.to_pylist()
    groups = {}
    for r in rows:
        groups.setdefault(tuple(r[k] for k in keys), []).append(r)
    out = {}
    for g in groups.values():
        for name, asc in reversed(list(presort.items())):
            nn = [r for r in g if r[name] is not None]
            nn.sort(key=lambda r: r[name], reverse=not asc)
            g = nn + [r for r in g if r[name] is None]
        for r, val in zip(g, fn(g)):
            out[r["rid"]] = val
    return [out[i] for i in range(len(rows))]


def _running(op, vals):
    res, acc, cnt = [], None, 0
    for x in vals:
        if x is not None:
            cnt += 1
            acc = x if acc is None else op(acc, x)
        res.append(acc)
    return res


def _wrap(v):
    return (v + (1 << 63)) % (1 << 64) - (1 << 63) if v is not None else None


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("presort", [OrderedDict(), OrderedDict(p=True), OrderedDict(p=False, v=True)])
def test_oracle_against_a_naive_per_group_loop(seed, presort):
    t = _table(300, seed)
    keys = ["k"]
    cols = [col("rid"), f.row_number().alias("rn"), f.rank().alias("rk"), f.dense_rank().alias("dr"),
            f.sum(col("v")).over(running=True).alias("rs"), f.sum(col("v")).over().alias("ts"),
            f.min(col("x")).over(running=True).alias("rmin"), f.max(col("v")).over().alias("tmax"),
            f.count(col("v")).over(running=True).alias("rc"), f.count(all_cols()).over().alias("n"),
            f.first(col("s")).over(running=True).alias("fs"), f.last(col("v")).over().alias("lv"),
            f.avg(col("v")).over().alias("av"), f.lag(col("s")).alias("lag"), f.lead(col("v"), 2, -1).alias("lead")]
    got = W.window_map(t, keys, presort, cols)
    pk = list(presort)

    def peers(g):
        return [tuple(r[k] for k in pk) for r in g]

    def rank(g, dense):
        out, pr = [], peers(g)
        d = 0
        for i, p in enumerate(pr):
            if i == 0 or p != pr[i - 1]:
                d += 1
                r = i + 1
            out.append(d if dense else r)
        return out

    def whole(fn):
        return lambda g: [fn(g)[-1]] * len(g)

    exp = {
        "rn": _naive(t, keys, presort, lambda g: list(range(1, len(g) + 1))),
        "rk": _naive(t, keys, presort, lambda g: rank(g, False)),
        "dr": _naive(t, keys, presort, lambda g: rank(g, True)),
        "rs": _naive(t, keys, presort, lambda g: _running(lambda a, b: a + b, [r["v"] for r in g])),
        "ts": _naive(t, keys, presort, whole(lambda g: _running(lambda a, b: a + b, [r["v"] for r in g]))),
        "rmin": _naive(t, keys, presort, lambda g: _running(min, [r["x"] for r in g])),
        "tmax": _naive(t, keys, presort, whole(lambda g: _running(max, [r["v"] for r in g]))),
        "rc": _naive(t, keys, presort, lambda g: list(np.cumsum([r["v"] is not None for r in g]))),
        "n": _naive(t, keys, presort, lambda g: [len(g)] * len(g)),
        "fs": _naive(t, keys, presort, lambda g: _running(lambda a, b: a, [r["s"] for r in g])),
        "lv": _naive(t, keys, presort, whole(lambda g: _running(lambda a, b: b, [r["v"] for r in g]))),
        "lag": _naive(t, keys, presort, lambda g: [None] + [r["s"] for r in g[:-1]]),
        "lead": _naive(t, keys, presort, lambda g: [r["v"] for r in g[2:]] + [-1] * min(2, len(g))),
    }
    for name, e in exp.items():
        assert got[name] == e, name
    sums = _naive(t, keys, presort, lambda g: [sum(r["v"] for r in g if r["v"] is not None)] * len(g))
    cnts = _naive(t, keys, presort, lambda g: [sum(r["v"] is not None for r in g)] * len(g))
    assert got["av"] == [s / c if c else None for s, c in zip(sums, cnts)]
    assert got["rid"] == list(range(t.num_rows))


def test_against_pandas_where_pandas_means_the_same():
    t = _table(2000, 7, nulls=False)
    df = t.to_pandas()
    keys, presort = ["k"], OrderedDict(p=True)
    got = W.window_map(t, keys, presort, [
        f.row_number().alias("rn"), f.lag(col("v"), 2).alias("lag2"), f.sum(col("v")).over(running=True).alias("cs"),
        f.sum(col("v")).over().alias("ts"), f.rank().alias("rk"), f.dense_rank().alias("dr")])
    srt = df.sort_values(["k", "p"], kind="stable")
    g = srt.groupby("k", sort=False)
    exp = pd.DataFrame({"rn": g.cumcount() + 1, "lag2": g["v"].shift(2), "cs": g["v"].cumsum(),
                        "ts": g["v"].transform("sum"), "rk": g["p"].rank(method="min"),
                        "dr": g["p"].rank(method="dense")}).sort_index()
    for c in ["rn", "cs", "ts", "rk", "dr"]:
        assert got[c] == exp[c].astype("int64").tolist(), c
    assert got["lag2"] == [None if pd.isna(x) else int(x) for x in exp["lag2"]]
    # running LAST over a column with NULLs is a per-group forward fill
    t2 = _table(2000, 8)
    d2 = t2.to_pandas()
    got = W.window_map(t2, ["k"], OrderedDict(), [f.last(col("x")).over(running=True).alias("ff")])
    exp = d2.groupby("k", dropna=False)["x"].ffill()
    assert got["ff"] == [None if pd.isna(x) else x for x in exp]


def _bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


def test_scan_wraps_int64_and_orders_floats_totally():
    off = np.array([0, 3, 3, 7], dtype=np.int64)
    big = np.iinfo(np.int64).max
    v, c = W.segmented_scan(np.array([big, 1, 1, 5, -2, 0, 3], dtype=np.int64), None, off, "SUM_I64")
    assert v.tolist() == [big, -big - 1, -big, 5, 3, 3, 6] and c.tolist() == [1, 2, 3, 1, 2, 3, 4]
    vals = [float("nan"), -0.0, 0.0, -math.inf, -float("nan"), 1.0, math.inf]
    bits = np.array([_bits(x) for x in vals], dtype=np.int64)
    bits[4] = _bits(float("nan")) | np.int64(-(1 << 63))  # -NaN
    one = np.array([0, 7], dtype=np.int64)
    lo, _ = W.segmented_scan(bits, None, one, "MIN_F64")
    hi, _ = W.segmented_scan(bits, None, one, "MAX_F64")
    assert lo.tolist() == [bits[0], bits[1], bits[1], bits[3], bits[4], bits[4], bits[4]]
    assert hi.tolist() == [bits[0]] * 7
    valid = np.array([0, 0, 1, 0, 1, 1, 0], dtype=bool)
    v, c = W.segmented_scan(np.arange(7, dtype=np.int64), valid, off, "MIN_I64")
    assert v.tolist() == [0, 0, 2, 0, 4, 4, 4] and c.tolist() == [0, 0, 1, 0, 1, 2, 2]
