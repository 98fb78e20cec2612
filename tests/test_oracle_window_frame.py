"""The moving-frame oracle (tests/_frame_oracle.py: ``frame_aggregate``, ``window_map`` with ``rows``) on CPU: the
vectorised form against the plain loop, trailing and centred frames against pandas ``groupby().rolling()``, and
the frames (None, 0) / (None, None) against the running and whole-partition results."""
from collections import OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from fugue_b200.column import all_cols, col, functions as f
from oracle import window as W

import _frame_oracle as F  # noqa: E402

OPS = ["COUNT", "SUM_I64", "SUM_F64", "MIN_I64", "MAX_I64", "MIN_F64", "MAX_F64"]
FRAMES = [(-2, 0), (-1, 1), (0, 0), (1, 3), (-5, -1), (None, -1), (None, 2), (0, None), (-3, None), (None, 0),
          (None, None), (-40, 40), (5, 7), (-2**63 + 1, 2**63 - 1), (2**63 - 1, 2**63 - 1)]


def _offsets(n: int, rng) -> np.ndarray:
    lens = np.minimum(rng.zipf(1.3, n), 60)
    lens[rng.random(n) < 0.05] = 0
    cut = np.concatenate([[0], np.cumsum(lens)])
    cut = cut[cut < n]
    return np.concatenate([cut, [n, n]]).astype(np.int64)


def _values(op: str, n: int, rng) -> np.ndarray:
    if op == "SUM_F64":  # multiples of 2^-10 below 2^20: every partial sum is exact
        return (rng.integers(-(2**30), 2**30, n) * 2.0 ** -10).view(np.int64)
    if op.endswith("F64"):
        special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, -1.5], dtype=np.float64)
        return np.where(rng.random(n) < 0.2, rng.choice(special, n), rng.standard_normal(n)).view(np.int64)
    return rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64, endpoint=True)


@pytest.mark.parametrize("op", OPS)
def test_vectorised_form_matches_the_loop(op):
    rng = np.random.default_rng(len(op))
    n = 2500
    off = _offsets(n, rng)
    v = _values(op, n, rng)
    m = rng.random(n) < 0.7
    m[off[1]:off[2]] = False  # an all-NULL segment
    for frame in FRAMES:
        for valid in (None, m):
            a = F.frame_aggregate(v, valid, off, op, *frame, loop=True)
            b = F.frame_aggregate(v, valid, off, op, *frame, loop=False)
            assert np.array_equal(a[1], b[1]), frame
            if op != "COUNT":
                assert np.array_equal(a[0], b[0]), frame


def test_the_loop_by_hand():
    off = np.array([0, 3, 3, 7], dtype=np.int64)
    v = np.array([1, 2, 3, 10, 20, 30, 40], dtype=np.int64)
    m = np.array([1, 1, 1, 1, 0, 1, 1], dtype=bool)
    r, c = F.frame_aggregate(v, m, off, "SUM_I64", -1, 0)
    assert r.tolist() == [1, 3, 5, 10, 10, 30, 70] and c.tolist() == [1, 2, 2, 1, 1, 1, 2]
    r, c = F.frame_aggregate(v, m, off, "MAX_I64", 1, 2)
    assert r.tolist() == [3, 3, 0, 30, 40, 40, 0] and c.tolist() == [2, 1, 0, 1, 2, 1, 0]
    _, c = F.frame_aggregate(None, None, off, "COUNT", -3, -1)
    assert c.tolist() == [0, 1, 2, 0, 1, 2, 3]
    r, c = F.frame_aggregate(v, m, off, "MIN_I64", 5, 7)
    assert r.tolist() == [0] * 7 and c.tolist() == [0] * 7


def test_f64_sum_adds_only_the_frame():
    v = np.array([1e20] + [1.0] * 50)
    for loop in (True, False):
        r, _ = F.frame_aggregate(v.view(np.int64), None, np.array([0, 51]), "SUM_F64", -2, 0, loop=loop)
        assert (r.view(np.float64)[3:] == 3.0).all()


def _series(n: int, rng):
    off = _offsets(n, rng)
    g = np.repeat(np.arange(len(off) - 1), np.diff(off))
    x = rng.standard_normal(n)
    ok = rng.random(n) < 0.8
    return off, g, x, ok


@pytest.mark.parametrize("w", [1, 3, 7, 30])
def test_trailing_and_centred_frames_match_pandas_rolling(w):
    rng = np.random.default_rng(w)
    n = 3000
    off, g, x, ok = _series(n, rng)
    s = pd.Series(np.where(ok, x, np.nan))
    for frame, center in [((-(w - 1), 0), False)] + ([((-(w // 2), w // 2), True)] if w % 2 == 1 else []):
        roll = s.groupby(g).rolling(w, min_periods=1, center=center)
        bits = x.view(np.int64)
        exp = {"SUM_F64": roll.sum(), "MIN_F64": roll.min(), "MAX_F64": roll.max(), "COUNT": roll.count()}
        for op, e in exp.items():
            e = e.reset_index(level=0, drop=True).sort_index().to_numpy()
            r, c = F.frame_aggregate(None if op == "COUNT" else bits, ok, off, op, *frame)
            if op == "COUNT":
                assert np.array_equal(c, e.astype(np.int64)), (op, frame)
                continue
            got = np.where(c > 0, r.view(np.float64), np.nan)
            if op == "SUM_F64":  # pandas keeps a running sum: compare with a tolerance
                assert np.allclose(got, e, rtol=1e-12, atol=1e-12, equal_nan=True), (op, frame)
            else:
                assert np.array_equal(got, e, equal_nan=True), (op, frame)
        mean = roll.mean().reset_index(level=0, drop=True).sort_index().to_numpy()
        r, c = F.frame_aggregate(bits, ok, off, "SUM_F64", *frame)
        assert np.allclose(np.where(c > 0, r.view(np.float64) / np.maximum(c, 1), np.nan), mean, rtol=1e-12,
                           atol=1e-12, equal_nan=True)


@pytest.mark.parametrize("op", OPS)
def test_unbounded_frames_are_the_running_and_whole_results(op):
    rng = np.random.default_rng(40 + len(op))
    n = 4000
    off = _offsets(n, rng)
    v = _values(op, n, rng)
    m = rng.random(n) < 0.6
    last = np.repeat(off[1:] - 1, np.diff(off))
    run_v, run_c = W.segmented_scan(v, m, off, op)
    for loop in (True, False):
        rv, rc = F.frame_aggregate(v, m, off, op, None, 0, loop=loop)
        wv, wc = F.frame_aggregate(v, m, off, op, None, None, loop=loop)
        assert np.array_equal(rc, run_c) and np.array_equal(wc, run_c[last])
        if op == "COUNT":
            continue
        if op == "SUM_F64" and loop:  # fsum vs a running sum: equal here, every partial sum is exact
            assert np.array_equal(rv.view(np.float64), run_v.view(np.float64))
        else:
            assert np.array_equal(rv, run_v) and np.array_equal(wv, run_v[last])


def test_window_map_with_frames():
    rng = np.random.default_rng(3)
    n = 600
    t = pa.table({"rid": np.arange(n), "k": pa.array(rng.integers(0, 7, n), mask=rng.random(n) < 0.05),
                  "p": rng.integers(0, 5, n), "v": pa.array(rng.integers(-50, 50, n), mask=rng.random(n) < 0.2),
                  "s": pa.array(list(np.array(["a", "b", "c"], dtype=object)[rng.integers(0, 3, n)]),
                                mask=rng.random(n) < 0.2, type=pa.string())})
    cols = [col("rid"), f.sum(col("v")).over(rows=(None, 0)).alias("a"), f.sum(col("v")).over(running=True).alias("b"),
            f.max(col("v")).over(rows=(None, None)).alias("c"), f.max(col("v")).over().alias("d"),
            f.sum(col("v")).over(rows=(-2, 0)).alias("m3"), f.count(all_cols()).over(rows=(1, 5)).alias("n5"),
            f.first(col("s")).over(rows=(-1, 1)).alias("fs"), (col("v") - f.avg(col("v")).over(rows=(-6, 0))).alias("dv")]
    out = F.window_map(t, ["k"], OrderedDict(p=True), cols)
    assert out["a"] == out["b"] and out["c"] == out["d"]
    # by hand from the oracle's partition order
    order = np.lexsort((np.arange(n), t.column("p").to_numpy(), t.column("k").is_null().to_numpy(),
                        t.column("k").fill_null(0).to_numpy()))
    pos = np.empty(n, dtype=np.int64)
    pos[order] = np.arange(n)
    key = [t.column("k")[int(i)].as_py() for i in order]
    v = [t.column("v")[int(i)].as_py() for i in order]
    for i in range(n):
        j = int(pos[i])
        frame = [v[q] for q in range(max(0, j - 2), j + 1) if key[q] == key[j] and v[q] is not None]
        assert out["m3"][i] == (sum(frame) if frame else None)
        assert out["n5"][i] == sum(1 for q in range(j + 1, min(n, j + 6)) if key[q] == key[j])
