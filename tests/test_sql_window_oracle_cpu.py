"""The reference of explicit windows (tests/_sql_window_oracle.py) checked against independent sources, without a GPU:
SQLite on int64 / float64 / string tables for every form of tests/test_sql_window_gpu.py, pandas on the float16 /
float32 / uint64 / date / timestamp columns SQLite cannot hold, and cases worked by hand (LAG / LEAD at n = 0, at the
partition length and at 2^63 - 1, NaN and -0.0 peers, a DESC RANGE frame on uint64 around 2^63).  Also the LAG / LEAD
default rule (DESIGN §7p): the oracle's plain-Python statement against ``colmap.offset_default``, value by value."""
import datetime
import math
import sqlite3
import struct
from collections import OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import _sql_window_oracle as O
import test_sql_window_gpu as SG
from fugue_b200.colmap import offset_default
from fugue_b200.sql import _parse_select
from oracle import window as W

I64_MAX = (1 << 63) - 1


def _items(text: str):
    return _parse_select(text, "FROM t", "SELECT " + text + " FROM t").columns


def _select(tbl: pa.Table, text: str) -> dict:
    out, keep = O.select(tbl, _items(text))
    assert keep == list(range(tbl.num_rows))
    return out


# ---- SQLite ------------------------------------------------------------------------------------------
def _against_sqlite(tbl: pa.Table, cases) -> None:
    out = _select(tbl, "rid, " + ", ".join(f"{d} AS w{i}" for i, (d, _) in enumerate(cases)))
    got = list(zip(*[out[k] for k in ["rid"] + [f"w{i}" for i in range(len(cases))]]))
    ref = ", ".join(f"{s or d} AS w{i}" for i, (d, s) in enumerate(cases))
    SG._same_rows(got, SG._sqlite(tbl, f"SELECT rid, {ref} FROM t ORDER BY rid"))


@pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 30), reason="needs SQLite >= 3.30")
@pytest.mark.parametrize("n,nkeys", [(0, 2), (1, 2), (2, 2), (300, 5), (2500, 3)])
def test_every_window_form_matches_sqlite(n, nkeys):
    _against_sqlite(SG._table(np.random.default_rng(n), n, nkeys=nkeys), SG.CASES)


@pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 30), reason="needs SQLite >= 3.30")
def test_all_null_keys_and_defaults_match_sqlite():
    tbl = SG._table(np.random.default_rng(11), 400, null_keys=True)
    cases = SG.CASES[:10] + [
        ("LEAD(vi, 400, 7) OVER (PARTITION BY ks ORDER BY t)", "LEAD(vi, 400, 7) OVER (PARTITION BY ks ORDER BY t NULLS LAST, rid)"),
        ("LAG(vf, 0) OVER (ORDER BY t)", "LAG(vf, 0) OVER (ORDER BY t NULLS LAST, rid)"),
        ("LAG(ks, 2, 'zz') OVER (PARTITION BY ki ORDER BY t DESC)",
         "LAG(ks, 2, 'zz') OVER (PARTITION BY ki ORDER BY t DESC NULLS LAST, rid)")]
    _against_sqlite(tbl, cases)


# ---- pandas ------------------------------------------------------------------------------------------
def _typed(rng, n: int, nan_as_null: bool = False) -> pa.Table:
    """Partition key k; float16 h and float32 f (multiples of 1/4, NaN, -0.0), uint64 u straddling 2^63 in steps that
    float64 holds exactly, date32 d and timestamp ts with a time zone, with NULLs.  ``nan_as_null``: pandas cannot
    tell a NaN from a NULL, so its rolling sums get NULLs only."""
    f = rng.integers(-40, 40, n) / 4.0
    f[rng.random(n) < 0.1] = np.nan
    f[rng.random(n) < 0.05] = -0.0
    u = (np.uint64(2**63) + (rng.integers(-20, 20, n) * 4096).astype(np.int64).astype(np.uint64))  # exact in float64
    days = rng.integers(-30, 30, n)
    return pa.table({
        "rid": np.arange(n, dtype=np.int64),
        "k": pa.array(rng.integers(0, 4, n), mask=rng.random(n) < 0.1, type=pa.int64()),
        "h": pa.array(f.astype(np.float16), from_pandas=nan_as_null),
        "f": pa.array(f.astype(np.float32), mask=(rng.random(n) < 0.05) | (nan_as_null & np.isnan(f))),
        "u": pa.array(u, type=pa.uint64()),
        "d": pa.array(days.astype(np.int32), mask=rng.random(n) < 0.05).cast(pa.date32()),
        "ts": pa.array(days * 3_600_000_000, mask=rng.random(n) < 0.05).cast(pa.timestamp("us", "Asia/Kolkata")),
    })


def _sorted_pdf(tbl: pa.Table, order: str, asc: bool) -> pd.DataFrame:
    pdf = tbl.to_pandas()
    pdf["h"] = pdf["h"].astype(np.float64)
    return pdf.sort_values(["k", order], ascending=[True, asc], kind="stable", na_position="last")


@pytest.mark.parametrize("order", ["h", "f", "u", "d", "ts"])
@pytest.mark.parametrize("asc", [True, False])
def test_ranks_match_pandas(order, asc):
    tbl = _typed(np.random.default_rng(1), 700)
    dirn = "" if asc else " DESC"
    out = _select(tbl, ", ".join(f"{fn}() OVER (PARTITION BY k ORDER BY {order}{dirn}) AS {fn}"
                                 for fn in ("ROW_NUMBER", "RANK", "DENSE_RANK")))
    pdf = tbl.to_pandas()
    pdf["h"] = pdf["h"].astype(np.float64)
    g = pdf.groupby(pdf["k"].fillna(-1), sort=False)[order]
    for fn, method in (("ROW_NUMBER", "first"), ("RANK", "min"), ("DENSE_RANK", "dense")):
        want = g.rank(method=method, ascending=asc, na_option="bottom").astype(np.int64).tolist()
        assert out[fn] == want, (fn, order, asc)


@pytest.mark.parametrize("n", [0, 1, 3, 60, 200, 10**6, I64_MAX])
@pytest.mark.parametrize("fn", ["LAG", "LEAD"])
def test_lag_lead_with_defaults_match_pandas_shift(fn, n):
    tbl = _typed(np.random.default_rng(2), 300)
    text = (f"{fn}(f, {n}, 0.5) OVER (PARTITION BY k ORDER BY d) AS f, {fn}(u, {n}, 18446744073709551615) OVER "
            f"(PARTITION BY k ORDER BY d) AS u, {fn}(d, {n}, DATE '2020-02-29') OVER (PARTITION BY k ORDER BY d) AS d, "
            f"{fn}(h, {n}, 65519.0) OVER (PARTITION BY k ORDER BY d) AS h")
    out = _select(tbl, text)
    pdf = _sorted_pdf(tbl, "d", True)
    shift = min(n, tbl.num_rows) * (1 if fn == "LAG" else -1)  # pandas takes n in int64: past the rows is the same
    g = pdf.groupby(pdf["k"].fillna(-1), sort=False)
    # 65519 rounds to 65504; dates as days since the epoch
    fills = {"f": 0.5, "u": 2**64 - 1, "d": (datetime.date(2020, 2, 29) - datetime.date(1970, 1, 1)).days, "h": 65504.0}
    for c, fill in fills.items():
        src = g["rid"].shift(shift)
        by_rid = dict(enumerate(O.storage_list(tbl[c])))  # Arrow's values: a NaN stays a NaN, a NULL is None
        want = {r: (fill if math.isnan(s) else by_rid[int(s)]) for r, s in zip(pdf["rid"].tolist(), src.tolist())}
        got = out[c]
        for r in range(tbl.num_rows):
            w = want[r]
            if isinstance(w, np.floating):
                w = float(w)
            assert got[r] == w or (isinstance(w, float) and math.isnan(w) and math.isnan(got[r])), (c, r, got[r], w)


@pytest.mark.parametrize("w", [1, 3, 40])
def test_rolling_sums_match_pandas(w):
    tbl = _typed(np.random.default_rng(3), 500, nan_as_null=True)
    out = _select(tbl, f"SUM(f) OVER (PARTITION BY k ORDER BY ts ROWS BETWEEN {w - 1} PRECEDING AND CURRENT ROW) AS s, "
                       f"SUM(h) OVER (PARTITION BY k ORDER BY u DESC ROWS {w - 1} PRECEDING) AS sh")
    for c, order, asc in (("f", "ts", True), ("h", "u", False)):
        pdf = _sorted_pdf(tbl, order, asc)
        x = pdf[c].astype(np.float64)
        r = x.groupby(pdf["k"].fillna(-1), sort=False).rolling(w, min_periods=1).sum()
        pdf["want"] = r.reset_index(level=0, drop=True)  # dyadic values: every partial sum is exact
        want = pdf.sort_values("rid")["want"].tolist()
        got = out["s" if c == "f" else "sh"]
        assert [None if isinstance(v, float) and math.isnan(v) else v for v in want] == got, c


# ---- by hand -------------------------------------------------------------------------------------------
def test_lag_lead_offsets_worked_by_hand():
    tbl = pa.table({"rid": [0, 1, 2, 3, 4], "k": [1, 2, 1, 1, 2], "v": pa.array([10, 20, None, 30, 40], pa.int8())})
    out = _select(tbl, "LAG(v, 0) OVER (PARTITION BY k ORDER BY rid) AS l0, "
                       "LEAD(v, 3, -1) OVER (PARTITION BY k ORDER BY rid) AS l3, "
                       "LAG(v, 2, 7) OVER (PARTITION BY k ORDER BY rid) AS l2, "
                       "LEAD(v, 9223372036854775807, 5) OVER (PARTITION BY k ORDER BY rid) AS big, "
                       "LAG(v, 9223372036854775807) OVER (ORDER BY rid) AS bignull, "
                       "LEAD(v, 1) OVER (PARTITION BY k ORDER BY rid DESC) AS d1")
    assert out["l0"] == [10, 20, None, 30, 40]
    assert out["l3"] == [-1, -1, -1, -1, -1]           # k=1 has 3 rows, k=2 has 2: n = 3 is past both
    assert out["l2"] == [7, 7, 7, 10, 7]
    assert out["big"] == [5, 5, 5, 5, 5]
    assert out["bignull"] == [None] * 5
    assert out["d1"] == [None, None, 10, None, 20]      # k=1 DESC: 3, 2, 0; k=2 DESC: 4, 1


def test_nan_and_signed_zero_are_peers_by_hand():
    nan_neg = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000001))[0]
    f = [0.0, -0.0, float("nan"), nan_neg, None, 1.0, -1.0]
    tbl = pa.table({"rid": list(range(7)), "f": pa.array(f, pa.float64())})
    out = _select(tbl, "RANK() OVER (ORDER BY f) AS r, DENSE_RANK() OVER (ORDER BY f DESC) AS dr, "
                       "COUNT(*) OVER (ORDER BY f) AS c, ROW_NUMBER() OVER (PARTITION BY f ORDER BY rid) AS rn")
    # ASC: -1 | 0, -0 | NaN, -NaN, NULL (all NULL)
    assert out["r"] == [2, 2, 5, 5, 5, 4, 1]
    assert out["c"] == [3, 3, 7, 7, 7, 4, 1]
    # DESC: 1 | 0, -0 | -1 | NULLs last
    assert out["dr"] == [2, 2, 4, 4, 4, 1, 3]
    assert out["rn"] == [1, 2, 1, 2, 3, 1, 1]


def test_desc_range_frame_on_uint64_around_2_63_by_hand():
    u = [2**63 - 2, 2**63 - 1, 2**63, 2**63 + 1, 2**63 + 3, 2**64 - 1, 0, None]
    tbl = pa.table({"rid": list(range(8)), "u": pa.array(u, pa.uint64())})
    out = _select(tbl, "COUNT(*) OVER (ORDER BY u DESC RANGE BETWEEN 2 PRECEDING AND 1 FOLLOWING) AS c, "
                       "MIN(rid) OVER (ORDER BY u DESC RANGE BETWEEN 1 PRECEDING AND CURRENT ROW) AS m")
    # DESC: row i's frame is the keys in [u_i - 1, u_i + 2]
    assert out["c"] == [3, 4, 3, 3, 1, 1, 1, 1]
    # keys in [u_i, u_i + 1]; the NULL key's frame is its NULL peers
    assert out["m"] == [0, 1, 2, 3, 4, 5, 6, 7]


# ---- the LAG / LEAD default rule ----------------------------------------------------------------------
_DEFAULT_TYPES = [pa.string(), pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(),
                  pa.float16(), pa.float32(), pa.float64(), pa.bool_(), pa.date32(), pa.date64(), pa.timestamp("s"),
                  pa.timestamp("ms"), pa.timestamp("us"), pa.timestamp("ns"), pa.timestamp("ms", "Asia/Kolkata")]
_DEFAULTS = [0, 1, -1, 127, 128, 255, 256, -129, 32767, 65535, 65536, 2**31, 2**32 - 1, 2**32, I64_MAX, 2**63,
             2**64 - 1, 2**64, -(2**63), -(2**63) - 1, 2.0, 2.5, -0.0, 0.1, 65519.0, 65520.0, 1e300, float("inf"),
             float("nan"), True, False, "x", datetime.date(2020, 2, 29), datetime.date(1, 1, 1),
             datetime.datetime(2020, 1, 1, 0, 0, 1), datetime.datetime(2020, 1, 1, 0, 0, 1, 500),
             datetime.datetime(2262, 4, 12), datetime.timedelta(days=1),
             # float16 values that rounding twice (through float32) gets wrong; an int past float64; aware timestamps
             65519.999, 1.0004883, 2049.0000001, -65519.999, 10**400,
             datetime.datetime(2020, 1, 1, 5, 30, tzinfo=datetime.timezone(datetime.timedelta(hours=5, minutes=30))),
             datetime.datetime(2020, 1, 1, 0, 0, 0, 1000, tzinfo=datetime.timezone.utc)]


@pytest.mark.parametrize("tp", _DEFAULT_TYPES, ids=str)
def test_default_rule_agrees_with_the_engine(tp):
    width = 0 if pa.types.is_string(tp) else 8 * {pa.bool_(): 1}.get(tp, max(tp.bit_width // 8, 1))
    for d in _DEFAULTS:
        try:
            want = W.offset_default(d, tp)
        except ValueError:
            with pytest.raises(ValueError):
                offset_default(d, tp, "LAG")
            continue
        got = offset_default(d, tp, "LAG")
        if pa.types.is_string(tp):
            assert got is None and want.to_pylist() == [d]
            continue
        raw = want.view({8: pa.uint8(), 16: pa.uint16(), 32: pa.uint32(), 64: pa.uint64()}[width]) \
            if not pa.types.is_boolean(tp) else pa.array([int(want[0].as_py())], pa.uint8())
        assert got == raw[0].as_py(), (tp, d, hex(got), raw)


def test_default_rule_by_hand():
    assert W.offset_default(0.5, pa.float16()).to_pylist() == [0.5]
    assert W.offset_default(2, pa.float16()).to_pylist() == [2.0]
    assert W.offset_default(2**64 - 1, pa.uint64()).to_pylist() == [2**64 - 1]
    assert W.offset_default(1e6, pa.float16()).to_pylist() == [math.inf]
    # once from float64 to half: 65519.999 is below the midpoint 65520 between 65504 and the overflow
    assert W.offset_default(65519.999, pa.float16()).to_pylist() == [65504.0]
    assert W.offset_default(2049.0000001, pa.float16()).to_pylist() == [2050.0]
    aware = datetime.datetime(2020, 1, 1, 5, 30, tzinfo=datetime.timezone(datetime.timedelta(hours=5, minutes=30)))
    assert W.offset_default(aware, pa.timestamp("s")).to_pylist() == [datetime.datetime(2020, 1, 1)]
    for d, tp in ((1000, pa.int8()), (2.5, pa.int64()), (2**64, pa.uint64()), (-1, pa.uint32()), ("x", pa.int64()),
                  (1, pa.bool_()), (5, pa.date32()), (datetime.datetime(2020, 1, 1, 12), pa.date32()),
                  (datetime.datetime(2020, 1, 1, 0, 0, 0, 500000), pa.timestamp("s")), (2, pa.string())):
        with pytest.raises(ValueError):
            W.offset_default(d, tp)
    # the oracle's window map applies it: LAG on a float16 column with a default of 0.5
    tbl = pa.table({"h": pa.array(np.array([1.0, 2.0], np.float16))})
    from fugue_b200.column import col, functions as f
    out = W.window_map(tbl, [], OrderedDict(), [f.lag(col("h"), 1, 0.5).alias("l")])
    assert out["l"] == [0.5, 1.0]
