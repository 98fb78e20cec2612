"""Window functions in SQL and ``select / assign / filter`` (DESIGN §7p) at every column type, against the exact reference
of tests/_sql_window_oracle.py: PARTITION BY and ORDER BY on each type and on expressions of them, window arguments of
each type under every frame kind, RANGE offsets on every orderable type (integer offsets at the int64 extremes and on
uint64 >= 2^63, float offsets beside infinities and NaN, INTERVAL offsets on dates and timestamps), LAG / LEAD with and
without defaults for n from 0 to 2^63 - 1, both ways back to input order at every output width, edge sizes around a K9
tile (2048 rows) and 2 M rows.

The types and values are those of tests/test_aggregate_routes_gpu.py: NULLs, the types' extremes, NaN of both signs
and with payloads, -0.0, infinities, uint64 at and above 2^63, non-ASCII strings.  Every test checks that rows come back
in input order and compares values bit for bit (floats by their bits, NaN payloads included); a float SUM / AVG is
compared exactly too, because its arguments are multiples of 1/4 that keep every partial sum exact; AVG of int64 and
uint64 within (m - 1) 2^-52 sum |x| / m of the exact mean."""
import struct
from typing import Any, Dict, List

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import _sql_window_oracle as O  # noqa: E402
import test_aggregate_routes_gpu as AR  # noqa: E402
from fugue_b200 import _lib  # noqa: E402
from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.sql import _parse_select  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402

DEV = torch.device("cuda", 0)
TYPES = AR.TYPES
NUMERIC = [nm for nm, tp in TYPES.items() if pa.types.is_integer(tp) or pa.types.is_floating(tp) or nm == "b"]
FLOATS = ("f16", "f32", "f64")
_ENGINE: List[Any] = []
I64_MAX = (1 << 63) - 1


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


# ---- the table -------------------------------------------------------------------------------------------
def _pooled(nm: str, n: int, rng: np.random.Generator, pool: int = 24):
    """Values of type ``nm`` drawn from a pool of ``pool`` edge-rich values, so that keys repeat; floats are multiples
    of 1/4 beside the type's finite edges (largest, smallest subnormal, +-0.0), +-inf and NaNs with payloads."""
    v, ok = AR._values(nm, "mixed", True, rng, pool)
    if nm in FLOATS:
        dt = v.dtype
        fin = (rng.integers(-64, 64, pool) / 4.0).astype(dt)
        edges, nonfin = AR._FLOAT_EDGES[nm]
        v = np.concatenate([fin, edges, np.array([0.0, -0.0], dt), nonfin])
        ok = np.concatenate([ok, np.ones(len(v) - len(ok), bool)])[:len(v)]
        ok[rng.random(len(v)) < 0.1] = False
    idx = rng.integers(0, len(v), n)
    return v[idx], ok[idx]


def _table(n: int, seed: int = 0, nkeys: int = 6) -> pa.Table:
    rng = np.random.default_rng(seed)
    cols: Dict[str, Any] = {"rid": pa.array(np.arange(n, dtype=np.int64))}
    cols["k"] = pa.array(rng.integers(0, nkeys, n), mask=rng.random(n) < 0.1, type=pa.int64())
    cols["o"] = pa.array(rng.integers(0, max(1, n // 3), n), mask=rng.random(n) < 0.05, type=pa.int64())
    cols["v"] = pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.1, type=pa.int64())
    cols["ff"] = pa.array(rng.integers(-9, 9, n) / 2.0, mask=rng.random(n) < 0.1, type=pa.float64())
    for nm in TYPES:
        v, ok = _pooled(nm, n, rng)
        cols[nm] = AR._arrow(nm, v, ok)
        if nm in FLOATS:  # for SUM / AVG: multiples of 1/4 only, so that every partial sum (and difference) is exact
            cols["p" + nm] = AR._arrow(nm, (rng.integers(-64, 64, n) / 4.0).astype(v.dtype), rng.random(n) > 0.1)
    return pa.table(cols)


# ---- running and comparing ----------------------------------------------------------------------------------
def _key(x: Any) -> Any:
    if isinstance(x, (float, np.floating)):
        return ("f", struct.unpack("<Q", struct.pack("<d", float(x)))[0])
    return x


def _device(tbl: pa.Table, items: str, rest: str = "") -> pa.Table:
    return fa.raw_sql(f"SELECT {items} FROM", _df(tbl), rest, engine=_engine(), as_fugue=True).as_arrow()


def _check(tbl: pa.Table, items: str, rest: str = "", qualify: str = None, skip=()) -> pa.Table:
    """The device's ``SELECT rid, items FROM tbl rest`` against the oracle, bit for bit; ``skip``: outputs the caller
    checks itself.  Returns the device's result."""
    got = _device(tbl, "rid, " + items, rest)
    cols = _parse_select("rid, " + items, "FROM t", "SELECT rid, " + items + " FROM t").columns
    q = None
    if qualify is not None:
        q = _parse_select("rid", f"FROM t QUALIFY {qualify}", f"SELECT rid FROM t QUALIFY {qualify}").qualify
    want, keep = O.select(tbl, cols, q)
    assert got["rid"].to_pylist() == keep  # rows keep their input order
    for nm in want:
        if nm in skip:
            continue
        g, w = O.storage_list(got[nm]), want[nm]
        bad = [i for i, (a, b) in enumerate(zip(g, w)) if _key(a) != _key(b)]
        assert len(g) == len(w) and not bad, (nm, [(i, g[i], w[i]) for i in bad[:5]])
    return got


# ---- PARTITION BY ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", list(TYPES) + ["UPPER(s)", "CAST(ff AS BIGINT)", "d32 + INTERVAL '1' DAY",
                                                "ts_ms - INTERVAL '1' DAY", "i64 % 3"])
def test_partition_by_each_type(key):
    tbl = _table(3000, seed=1)
    _check(tbl, f"ROW_NUMBER() OVER (PARTITION BY {key} ORDER BY o) AS rn, COUNT(*) OVER (PARTITION BY {key}) AS c, "
                f"SUM(v) OVER (PARTITION BY {key}) AS s, LAG(rid) OVER (PARTITION BY {key} ORDER BY o) AS lg")


# ---- ORDER BY ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("asc", ["ASC", "DESC"])
@pytest.mark.parametrize("key", list(TYPES))
def test_order_by_each_type(key, asc):
    tbl = _table(2600, seed=2)
    spec = f"(PARTITION BY k ORDER BY {key} {asc})"
    _check(tbl, f"ROW_NUMBER() OVER {spec} AS rn, RANK() OVER {spec} AS r, DENSE_RANK() OVER {spec} AS dr, "
                f"LAG(rid) OVER {spec} AS lg, LEAD(rid, 2) OVER {spec} AS ld, COUNT(*) OVER {spec} AS c, "
                f"SUM(v) OVER {spec} AS s")


@pytest.mark.parametrize("spec", ["(PARTITION BY k ORDER BY f32 DESC, s)", "(ORDER BY d64, u64 DESC, b)",
                                  "(PARTITION BY f64 ORDER BY f64 DESC, i16)", "(PARTITION BY k, s ORDER BY k DESC, ts_ns)",
                                  "(PARTITION BY ts_tz ORDER BY ts_tz DESC)",
                                  # one order value over the whole table: only the partition starts split the peers
                                  "(PARTITION BY f16 ORDER BY rid * 0)", "(PARTITION BY k ORDER BY rid % 1 DESC)"])
def test_several_order_keys_and_a_partition_key_in_order_by(spec):
    tbl = _table(3000, seed=3)
    _check(tbl, f"ROW_NUMBER() OVER {spec} AS rn, RANK() OVER {spec} AS r, DENSE_RANK() OVER {spec} AS dr, "
                f"COUNT(*) OVER {spec} AS c, LAG(rid, 1, -1) OVER {spec} AS lg")


# ---- window arguments ------------------------------------------------------------------------------------------
FRAMES = {"whole": "(PARTITION BY k)", "running": "(PARTITION BY k ORDER BY o ROWS UNBOUNDED PRECEDING)",
          "rows": "(PARTITION BY k ORDER BY o ROWS BETWEEN 3 PRECEDING AND 2 FOLLOWING)",
          "rows_wide": "(PARTITION BY k ORDER BY o ROWS BETWEEN 1500 PRECEDING AND 10 FOLLOWING)",
          "range": "(PARTITION BY k ORDER BY o RANGE BETWEEN 40 PRECEDING AND 25 FOLLOWING)",
          "default": "(PARTITION BY k ORDER BY o DESC)"}


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("arg", list(TYPES))
def test_window_arguments_of_each_type(arg, frame):
    tbl = _table(6000, seed=4, nkeys=3)  # partitions of ~2000 rows: the wide frame runs the combine path
    w = FRAMES[frame]
    heads = ["FIRST", "LAST", "COUNT"] + ([] if arg == "s" else ["MIN", "MAX"])  # strings: tests/test_strings_gpu.py
    items = [f"{h}({arg}) OVER {w} AS {h.lower()}" for h in heads]
    if arg in NUMERIC:
        summed = "p" + arg if arg in FLOATS else arg
        items += [f"SUM({summed}) OVER {w} AS sum", f"AVG({summed}) OVER {w} AS avg"]
    if frame == "whole":
        items += [f"LAG({arg}) OVER (PARTITION BY k ORDER BY o) AS lag",
                  f"LEAD({arg}, 3) OVER (PARTITION BY k ORDER BY o) AS lead"]
    wide = arg in ("i64", "u64")  # float64 sums of these are inexact: AVG within its bound
    got = _check(tbl, ", ".join(items), skip=("avg",) if wide else ())
    if wide:
        _check_wide_avg(tbl, arg, w, got["avg"].to_pylist())


def _check_wide_avg(tbl: pa.Table, arg: str, w: str, got: List[Any]) -> None:
    """AVG of an int64 / uint64 column (uint64 as its int64 bit pattern, §7e) over frame ``w``: the values become
    doubles d, whose exact frame sum S and sum of |d| the reference gives as 32-bit halves (int64 sums that cannot
    wrap).  The device's mean is within ``(m - 1) 2^-52 sum |d| / m`` of float(S) / m, plus one rounding of the
    quotient, as in tests/test_aggregate_routes_gpu.py."""
    x = tbl[arg].combine_chunks()
    vals = (x.view(pa.int64()) if arg == "u64" else x).to_pylist()
    d = [None if v is None else int(float(v)) for v in vals]  # float(v) is an integer of at most 2^63
    parts = {"h": [None if v is None else v >> 32 for v in d], "l": [None if v is None else v & 0xFFFFFFFF for v in d],
             "ah": [None if v is None else abs(v) >> 32 for v in d],
             "al": [None if v is None else abs(v) & 0xFFFFFFFF for v in d]}
    aux = tbl.select(["rid", "k", "o"])
    for nm, c in parts.items():
        aux = aux.append_column(nm, pa.array(c, type=pa.int64()))
    items = ", ".join(f"SUM({nm}) OVER {w} AS {nm}" for nm in parts) + f", COUNT(h) OVER {w} AS m"
    ref, _ = O.select(aux, _parse_select(items, "FROM t", "SELECT " + items + " FROM t").columns)
    for i, g in enumerate(got):
        m = ref["m"][i]
        if m == 0:
            assert g is None, (i, g)
            continue
        want = float(ref["h"][i] * 2**32 + ref["l"][i]) / m
        bound = (m - 1) * 2.0 ** -52 * float(ref["ah"][i] * 2**32 + ref["al"][i]) / m + 2.0 ** -52 * abs(want)
        assert g is not None and abs(g - want) <= bound, (i, g, want, bound)


# ---- RANGE offsets --------------------------------------------------------------------------------------------
_UNIT_PER_HOUR = {"ts_s": 3600, "ts_ms": 3_600_000, "ts_us": 3_600_000_000, "ts_ns": 3_600_000_000_000,
                  "ts_tz": 3_600_000, "d32": None, "d64": None}


def _range_table(nm: str, n: int, seed: int) -> pa.Table:
    """A key of type ``nm`` whose values lie close enough for frames of several rows, with the type's extremes."""
    rng = np.random.default_rng(seed)
    tp = TYPES[nm]
    ok = rng.random(n) > 0.08
    if nm in FLOATS:
        v = (rng.integers(-40, 40, n) / 4.0)
        edge = rng.random(n) < 0.1
        v[edge] = rng.choice(np.array([np.inf, -np.inf, np.nan, -np.nan, -0.0]), int(edge.sum()))
        key = pa.array(v.astype(AR._FLOAT_EDGES[nm][0].dtype), mask=~ok)
    elif nm in AR._NP:
        info = np.iinfo(AR._NP[nm])
        near = [int(info.min), int(info.min) + 3, int(info.max) - 2, int(info.max), 0, 5, 9]
        if nm == "u64":
            near += [2**63 - 2, 2**63, 2**63 + 1, 2**63 + 4]
        elif nm == "i64":
            near += [-3, 2]
        v = [near[i] + int(d) if info.min <= near[i] + int(d) <= info.max else near[i]
             for i, d in zip(rng.integers(0, len(near), n).tolist(), rng.integers(-3, 4, n))]
        key = pa.array([x if o else None for x, o in zip(v, ok.tolist())], type=tp)
    elif nm in ("d32", "d64"):
        days = rng.integers(-20, 20, n)
        key = pa.array(days.astype(np.int32), mask=~ok).cast(pa.date32())
        key = key if nm == "d32" else key.cast(pa.date64())
    else:
        hours = rng.integers(-60, 60, n) * _UNIT_PER_HOUR[nm] // 2  # half hours
        key = pa.array(hours, mask=~ok, type=pa.int64()).view(tp)
    return pa.table({"rid": np.arange(n, dtype=np.int64), "k": pa.array(rng.integers(0, 3, n)), "x": key,
                     "v": pa.array(rng.integers(-100, 100, n))})


def _offsets(nm: str) -> List[str]:
    if nm in FLOATS:
        return ["RANGE BETWEEN 1.5 PRECEDING AND 0.25 FOLLOWING", "RANGE BETWEEN 0.5 FOLLOWING AND 3 FOLLOWING"]
    if nm in ("d32", "d64"):
        return ["RANGE BETWEEN INTERVAL '2' DAY PRECEDING AND INTERVAL '1' DAY FOLLOWING",
                "RANGE BETWEEN INTERVAL '3' DAY PRECEDING AND INTERVAL '1' DAY PRECEDING"]
    if nm.startswith("ts"):
        return ["RANGE BETWEEN INTERVAL '0 01:30:00' DAY TO SECOND PRECEDING AND INTERVAL '0 00:30:00' DAY TO SECOND FOLLOWING",
                "RANGE BETWEEN INTERVAL '1' HOUR FOLLOWING AND UNBOUNDED FOLLOWING"]
    return ["RANGE BETWEEN 3 PRECEDING AND 2 FOLLOWING", "RANGE BETWEEN 2 FOLLOWING AND 6 FOLLOWING",
            "RANGE BETWEEN UNBOUNDED PRECEDING AND 1 PRECEDING"]


@pytest.mark.parametrize("asc", ["ASC", "DESC"])
@pytest.mark.parametrize("nm", [nm for nm in TYPES if nm not in ("b", "s")])
def test_range_offsets_on_each_type(nm, asc):
    tbl = _range_table(nm, 2500, seed=5)
    items = []
    for i, fr in enumerate(_offsets(nm)):
        w = f"(PARTITION BY k ORDER BY x {asc} {fr})"
        items += [f"COUNT(*) OVER {w} AS c{i}", f"SUM(v) OVER {w} AS s{i}", f"MIN(rid) OVER {w} AS m{i}",
                  f"LAST(x) OVER {w} AS l{i}"]
    _check(tbl, ", ".join(items))


@pytest.mark.parametrize("nm,frame", [
    ("i32", "RANGE BETWEEN INTERVAL '1' DAY PRECEDING AND CURRENT ROW"),
    ("u64", "RANGE BETWEEN INTERVAL '1' DAY PRECEDING AND CURRENT ROW"),
    ("d32", "RANGE BETWEEN INTERVAL '36' HOUR PRECEDING AND CURRENT ROW"),
    ("ts_s", "RANGE BETWEEN INTERVAL '0.5' SECOND PRECEDING AND CURRENT ROW"),
    ("i64", "RANGE BETWEEN 1.5 PRECEDING AND CURRENT ROW"),
    ("u8", "RANGE BETWEEN CURRENT ROW AND 0.5 FOLLOWING"),
])
def test_range_offsets_the_key_cannot_take_are_rejected(nm, frame):
    tbl = _range_table(nm, 50, seed=6)
    with pytest.raises(ValueError):
        _device(tbl, f"rid, COUNT(*) OVER (ORDER BY x {frame}) AS c")


# ---- LAG / LEAD defaults -------------------------------------------------------------------------------------
DEFAULTS = {"i8": "-128", "i16": "32767", "i32": "-7", "i64": "-9223372036854775808", "u8": "255", "u16": "65535",
            "u32": "4294967295", "u64": "18446744073709551615", "f16": "0.5", "f32": "0.1", "f64": "-0.0", "b": "TRUE",
            "d32": "DATE '2020-02-29'", "d64": "DATE '1900-01-01'", "ts_s": "TIMESTAMP '2020-01-01 00:00:01'",
            "ts_ms": "TIMESTAMP '1960-01-01 00:00:00.123'", "ts_us": "TIMESTAMP '2020-01-01 00:00:00.000001'",
            "ts_ns": "DATE '2000-01-01'", "ts_tz": "TIMESTAMP '2020-01-01 05:30:00'", "s": "'日本語'"}


@pytest.mark.parametrize("nm", list(TYPES))
def test_lag_lead_defaults_on_each_type(nm):
    tbl = _table(2200, seed=7, nkeys=4)
    items = []
    for i, n in enumerate([0, 1, 7, 600, 2200, 10**9, I64_MAX]):
        w = "(PARTITION BY k ORDER BY o)"
        items += [f"LAG({nm}, {n}, {DEFAULTS[nm]}) OVER {w} AS lag{i}", f"LEAD({nm}, {n}, {DEFAULTS[nm]}) OVER {w} AS lead{i}",
                  f"LEAD({nm}, {n}) OVER {w} AS bare{i}"]
    _check(tbl, ", ".join(items))


@pytest.mark.parametrize("item", ["LAG(f16, 1, 2) OVER (ORDER BY o)", "LEAD(f16, 1, 65519.0) OVER (ORDER BY o)",
                                  # rounded twice (through float32) these give +inf and 2048
                                  "LEAD(f16, 1, 65519.999) OVER (ORDER BY o)",
                                  "LAG(f16, 2, 2049.0000001) OVER (PARTITION BY k ORDER BY o)",
                                  "LAG(f32, 3, 16777217) OVER (PARTITION BY k ORDER BY o)"])
def test_float_defaults_round_to_nearest(item):
    _check(_table(500, seed=8), item + " AS w")


@pytest.mark.parametrize("item", ["LAG(i8, 1, 1000)", "LAG(i64, 1, 2.5)", "LEAD(u64, 1, -1)", "LAG(u32, 1, 4294967296)",
                                  "LAG(d32, 1, TIMESTAMP '2020-01-01 12:00:00')", "LAG(ts_s, 1, TIMESTAMP '2020-01-01 00:00:00.5')",
                                  "LAG(i32, 1, 'x')", "LAG(s, 1, 3)", "LAG(b, 1, 1)", "LAG(d64, 1, 5)"])
def test_defaults_the_type_cannot_hold_are_rejected(item):
    with pytest.raises(ValueError):
        _device(_table(50, seed=9), f"rid, {item} OVER (PARTITION BY k ORDER BY o) AS w")


# ---- back to input order: both paths ---------------------------------------------------------------------------
class _Spy:
    def __init__(self, monkeypatch: Any):
        lib = _lib.load()
        self.scatters: List[int] = []
        real = lib.fb_scatter_rows

        def spy(*a: Any) -> int:
            self.scatters.append(int(a[2]))
            return real(*a)

        monkeypatch.setattr(lib, "fb_scatter_rows", spy)


@pytest.mark.parametrize("nm", ["i8", "b", "i16", "f16", "i32", "f32", "d32", "i64", "u64", "f64", "ts_ns", "s"])
def test_one_window_per_spec_scatters_and_more_gather(nm, monkeypatch):
    tbl = _table(5000, seed=10)
    spy = _Spy(monkeypatch)
    # one output per spec: fb_scatter_rows, with a validity column (LAG) and without one (ROW_NUMBER)
    _check(tbl, f"LAG({nm}) OVER (PARTITION BY k ORDER BY o) AS a")
    assert spy.scatters == [1]
    spy.scatters.clear()
    _check(tbl, f"ROW_NUMBER() OVER (PARTITION BY {nm} ORDER BY o DESC) AS a")
    assert spy.scatters == [1]
    spy.scatters.clear()
    # two and three outputs of mixed widths: the inverse permutation and one gather, no scatter
    _check(tbl, f"FIRST({nm}) OVER (PARTITION BY k ORDER BY o) AS a, LEAD(i8, 2) OVER (PARTITION BY k ORDER BY o) AS b")
    _check(tbl, f"LAST({nm}) OVER (PARTITION BY i16 ORDER BY o) AS a, RANK() OVER (PARTITION BY i16 ORDER BY o) AS b, "
                f"LAG(s) OVER (PARTITION BY i16 ORDER BY o) AS c")
    assert spy.scatters == []


# ---- sizes -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 2, 2047, 2048, 2049, 5 * 2048 + 3])
def test_edge_sizes(n):
    tbl = _table(n, seed=n, nkeys=2)  # two partitions: each spans K9 tiles from 4096 rows
    _check(tbl, "ROW_NUMBER() OVER (PARTITION BY k ORDER BY f32 DESC) AS rn, RANK() OVER (PARTITION BY u64 ORDER BY d32) "
                "AS r, SUM(v) OVER (PARTITION BY k ORDER BY o) AS s, MAX(f64) OVER (PARTITION BY k ORDER BY o ROWS BETWEEN "
                "1100 PRECEDING AND 3 FOLLOWING) AS mx, LAG(s, 3, 'zz') OVER (PARTITION BY b ORDER BY ts_ns) AS lg, "
                "COUNT(i8) OVER (PARTITION BY k ORDER BY i32 RANGE BETWEEN 100000 PRECEDING AND CURRENT ROW) AS c")


def test_two_million_rows_against_pandas():
    rng = np.random.default_rng(12)
    n = 2_000_000
    h = (rng.integers(-64, 64, n) / 4.0).astype(np.float16)
    h[rng.random(n) < 0.01] = np.float16(-0.0)
    u = np.uint64(2**63) + (rng.integers(-1000, 1000, n) * 4096).astype(np.int64).astype(np.uint64)
    tbl = pa.table({"rid": np.arange(n, dtype=np.int64), "k": pa.array(rng.integers(0, 500, n), type=pa.uint64()),
                    "u": pa.array(u), "h": pa.array(h), "v": rng.integers(-1000, 1000, n)})
    got = _device(tbl, "rid, RANK() OVER (PARTITION BY k ORDER BY u DESC) AS r, LAG(h, 2, 0.5) OVER (PARTITION BY k "
                       "ORDER BY u DESC) AS lg, SUM(v) OVER (PARTITION BY h) AS s").to_pandas()
    pdf = tbl.to_pandas()
    pdf["h"] = pdf["h"].astype(np.float64)
    assert np.array_equal(got["rid"].to_numpy(), np.arange(n))
    g = pdf.groupby("k", sort=False)["u"]
    assert np.array_equal(got["r"].to_numpy(), g.rank(method="min", ascending=False).astype(np.int64).to_numpy())
    srt = pdf.sort_values(["k", "u"], ascending=[True, False], kind="stable")
    lag = srt.groupby("k", sort=False)["h"].shift(2, fill_value=0.5)
    want = lag.sort_index().to_numpy()
    assert np.array_equal(got["lg"].to_numpy(dtype=np.float64), want)
    assert np.array_equal(got["s"].to_numpy(), pdf.groupby("h")["v"].transform("sum").to_numpy())  # -0.0 joins 0.0


# ---- around the windows ---------------------------------------------------------------------------------------------
def test_several_specs_and_qualify_on_typed_windows():
    tbl = _table(4000, seed=13)
    items = ("RANK() OVER (PARTITION BY f16 ORDER BY u64 DESC) AS r, MAX(d64) OVER (PARTITION BY s) AS md, "
             "LEAD(ts_tz, 1) OVER (PARTITION BY k ORDER BY i8) AS ld, COUNT(*) OVER (PARTITION BY b ORDER BY f32) AS c, "
             "v * 2 - SUM(v) OVER (PARTITION BY u16 % 3) AS e")
    _check(tbl, items)
    _check(tbl, "RANK() OVER (PARTITION BY f16 ORDER BY u64 DESC) AS r",
           "QUALIFY RANK() OVER (PARTITION BY f16 ORDER BY u64 DESC) <= 2",
           qualify="RANK() OVER (PARTITION BY f16 ORDER BY u64 DESC) <= 2")


@pytest.mark.parametrize("key", ["f64", "f32", "u64", "s", "d32"])
def test_windows_over_group_by_results(key):
    tbl = _table(6000, seed=14)
    got = _device(tbl, f"{key}, SUM(v) AS sv, RANK() OVER (ORDER BY SUM(v) DESC) AS r, LAG(SUM(v)) OVER "
                       f"(ORDER BY {key}) AS p, SUM(COUNT(*)) OVER () AS n, COUNT(*) OVER () AS g, COUNT(*) OVER "
                       f"(PARTITION BY SUM(v) > 0) AS gp", f"GROUP BY {key}")

    def group(x: Any) -> Any:  # NaN of every sign and payload is one NULL group with the NULLs, -0.0 joins 0.0
        return None if x is None or x != x else (x + 0.0 if isinstance(x, float) else x)

    sums: Dict[Any, Any] = {}
    for x, v in zip(O.storage_list(tbl[key]), tbl["v"].to_pylist()):
        s = sums.setdefault(group(x), None)
        sums[group(x)] = s if v is None else (s or 0) + v
    keys = O.storage_list(got[key])
    assert sorted(map(repr, map(group, keys))) == sorted(map(repr, sums))
    assert got["sv"].to_pylist() == [sums[group(x)] for x in keys]
    assert got["g"].to_pylist() == [len(keys)] * len(keys)
    pos = [None if s is None else s > 0 for s in got["sv"].to_pylist()]
    assert got["gp"].to_pylist() == [pos.count(p) for p in pos]
    grouped = pa.table({"g": got[key], "s": got["sv"],
                        "rid": np.arange(len(keys), dtype=np.int64)})
    items = "RANK() OVER (ORDER BY s DESC) AS r, LAG(s) OVER (ORDER BY g) AS p"
    want, _ = O.select(grouped, _parse_select(items, "FROM t", "SELECT " + items + " FROM t").columns)
    assert got["r"].to_pylist() == want["r"] and got["p"].to_pylist() == want["p"]
    assert got["n"].to_pylist() == [tbl.num_rows] * len(keys)


def test_builder_nodes_equal_the_sql_text():
    tbl = _table(3000, seed=15)
    rn = f.rank().over(partition_by=[col("f16")], order_by=[("u64", False)])
    lg = f.lag(col("f16"), 2, 0.5).over(partition_by=["k"], order_by=["d32"])
    mx = f.max(col("ts_tz")).over(rows=(-3, 1), partition_by=[col("s")], order_by=["o"])
    sql = _check(tbl, "RANK() OVER (PARTITION BY f16 ORDER BY u64 DESC) AS rn, LAG(f16, 2, 0.5) OVER (PARTITION BY k "
                      "ORDER BY d32) AS lg, MAX(ts_tz) OVER (PARTITION BY s ORDER BY o ROWS BETWEEN 3 PRECEDING AND 1 "
                      "FOLLOWING) AS mx")
    def same(a: pa.Table, b: pa.Table) -> bool:
        return a.column_names == b.column_names and all(
            [_key(x) for x in O.storage_list(a[c])] == [_key(x) for x in O.storage_list(b[c])] for c in a.column_names)

    sel = fa.select(_df(tbl), "rid", rn.alias("rn"), lg.alias("lg"), mx.alias("mx"), engine=_engine(),
                    as_fugue=True).as_arrow()
    assert same(sel, sql)
    asg = fa.assign(_df(tbl), rn=rn, lg=lg, mx=mx, engine=_engine(), as_fugue=True).as_arrow()
    assert same(asg.select(["rid", "rn", "lg", "mx"]), sql)
    flt = fa.filter(_df(tbl), rn == 1, engine=_engine(), as_fugue=True).as_arrow()
    assert flt["rid"].to_pylist() == [r for r, x in zip(sql["rid"].to_pylist(), sql["rn"].to_pylist()) if x == 1]
