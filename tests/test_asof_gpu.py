"""As-of joins on the H100 (DESIGN §7q): ``fa.asof_join`` against ``oracle.asof`` row by row in left order, at edge
sizes, on every as-of type with NULLs / NaN / -0.0 / uint64 >= 2^63, at the int64 extremes with a tolerance, on
integer / float / string / two-column keys (a weak surrogate hash included), inner and left outer; against
``pandas.merge_asof`` through ``fa.asof_join`` and ``fa.raw_sql``; and ``fb_asof_search`` alone against
``numpy.searchsorted``."""
import datetime
from typing import Any, List

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from oracle import asof as A

DEV = torch.device("cuda", 0)
_ENGINE: List[Any] = []
DIRS = [(d, x) for d in A.DIRECTIONS for x in (True, False)]


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _device(left: pa.Table, right: pa.Table, on, asof, **kw) -> pa.Table:
    return fa.asof_join(left, right, on=on, asof=asof, engine=_engine(), as_fugue=True, **kw).as_arrow()


def _check(left: pa.Table, right: pa.Table, on, asof, how="left_outer", direction="backward", exact=True, tol=None,
           tol_units=None):
    """The device against the oracle on a right side that carries its row number in ``rid``."""
    got = _device(left, right, on, asof, how=how, direction=direction, allow_exact_matches=exact, tolerance=tol)
    exp = A.asof_join(left, right, on, asof, how, direction, exact, tol if tol_units is None else tol_units)
    assert got.column_names == exp.column_names
    for n in exp.column_names:
        a, b = got.column(n).to_pylist(), exp.column(n).to_pylist()
        assert a == b or _same_floats(a, b), (n, direction, exact, tol)
    return got


def _same_floats(a, b) -> bool:
    return len(a) == len(b) and all(x == y or (x != x and y != y) for x, y in zip(a, b))


def _numpy_match(lk, lt, rk, rt, direction="backward", exact=True, tol=None, lok=None, rok=None):
    n1, n2 = len(lk), len(rk)
    return A.match_rows_np(lk, lt, np.ones(n1, bool) if lok is None else lok, rk, rt,
                           np.ones(n2, bool) if rok is None else rok, direction, exact, tol)


def _rid(got: pa.Table) -> np.ndarray:
    return got.column("rid").fill_null(-1).to_numpy()


@pytest.mark.parametrize("n1,n2", [(0, 0), (0, 5), (5, 0), (1, 1), (1, 3), (3, 1), (2047, 2049), (2049, 2047),
                                   (4095, 4097), (4097, 1)])
@pytest.mark.parametrize("direction,exact", DIRS)
def test_edge_sizes(n1, n2, direction, exact):
    rng = np.random.default_rng(n1 * 7 + n2)
    left = pa.table({"k": rng.integers(0, 9, n1), "t": rng.integers(0, 300, n1), "v": rng.standard_normal(n1)})
    right = pa.table({"k": rng.integers(0, 8, n2), "t": rng.integers(0, 300, n2), "rid": np.arange(n2)})
    _check(left, right, ["k"], "t", "left_outer", direction, exact)
    _check(left, right, ["k"], "t", "inner", direction, exact)
    _check(left, right.drop(["k"]), [], "t", "inner", direction, exact, tol=7)


def test_one_long_run():
    """One key whose run holds 10^6 right rows."""
    rng = np.random.default_rng(1)
    n1, n2 = 300_000, 1_000_000
    lt, rt = rng.integers(-10, 3_000_010, n1), rng.integers(0, 3_000_000, n2)
    left = pa.table({"k": np.full(n1, 5), "t": lt})
    right = pa.table({"k": np.full(n2, 5), "t": rt, "rid": np.arange(n2)})
    for direction, exact in DIRS:
        got = _device(left, right, ["k"], "t", how="left_outer", direction=direction, allow_exact_matches=exact)
        exp = _numpy_match(np.full(n1, 5), lt, np.full(n2, 5), rt, direction, exact)
        assert np.array_equal(_rid(got), exp), (direction, exact)


@pytest.mark.parametrize("how", ["inner", "left_outer"])
def test_ten_million_left_rows(how):
    """10^7 left x 10^6 right rows with 65 536 keys."""
    rng = np.random.default_rng(2)
    n1, n2, nk = 10_000_000, 1_000_000, 65_536
    lk, rk = rng.integers(0, nk + 100, n1), rng.integers(0, nk, n2)
    lt, rt = rng.integers(0, 1 << 40, n1), rng.integers(0, 1 << 40, n2)
    left = pa.table({"k": lk, "t": pa.array(lt, pa.timestamp("us")), "v": rng.standard_normal(n1)})
    right = pa.table({"k": rk, "t": pa.array(rt, pa.timestamp("us")), "rid": np.arange(n2)})
    got = _device(left, right, ["k"], "t", how=how)
    exp = _numpy_match(lk, lt, rk, rt)
    keep = np.arange(n1) if how == "left_outer" else np.flatnonzero(exp >= 0)
    assert got.num_rows == len(keep)
    assert np.array_equal(got.column("k").to_numpy(), lk[keep])
    assert np.array_equal(got.column("v").to_numpy(), left.column("v").to_numpy()[keep])
    assert np.array_equal(_rid(got), exp[keep])


_INTS = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64()]
_TEMPORAL = [pa.date32(), pa.date64(), pa.timestamp("s"), pa.timestamp("ns", "UTC"), pa.duration("ms"),
             pa.time64("us")]
_FLOATS = [pa.float16(), pa.float32(), pa.float64()]


def _values(tp: pa.DataType, n: int, rng: np.random.Generator) -> pa.Array:
    """n values of ``tp`` with NULLs, few distinct values (ties), and the type's edge values."""
    mask = rng.random(n) < 0.1
    if tp in _FLOATS:
        base = rng.integers(-40, 40, n).astype(np.float64) / 4
        specials = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf], np.float64)
        pick = rng.random(n) < 0.15
        base[pick] = specials[rng.integers(0, len(specials), int(pick.sum()))]
        return pa.array(base.astype(tp.to_pandas_dtype()), tp, mask=mask)
    if tp == pa.uint64():
        v = rng.integers(0, 60, n).astype(np.uint64) + np.uint64((1 << 63) - 30)  # straddles 2^63
        v[rng.random(n) < 0.05] = np.uint64((1 << 64) - 1)
        return pa.array(v, tp, mask=mask)
    if tp in _INTS:
        info = np.iinfo(tp.to_pandas_dtype())
        v = rng.integers(-40, 40, n) if info.min < 0 else rng.integers(0, 80, n)
        v = v.astype(np.int64)
        v[rng.random(n) < 0.05] = info.max
        v[rng.random(n) < 0.05] = info.min
        return pa.array(v.astype(tp.to_pandas_dtype()), tp, mask=mask)
    storage = pa.int32() if tp == pa.date32() else pa.int64()
    v = rng.integers(0, 80, n) * (1 if tp == pa.date32() else 1000)
    return pa.array(v, storage, mask=mask).cast(tp) if tp != pa.time64("us") else \
        pa.array(v % 86_400_000_000, storage, mask=mask).view(tp)


@pytest.mark.parametrize("tp", _INTS + _FLOATS + _TEMPORAL, ids=str)
@pytest.mark.parametrize("direction,exact", DIRS)
def test_every_asof_type(tp, direction, exact):
    rng = np.random.default_rng(len(str(tp)) * 31 + len(direction) + exact)
    n1, n2 = 700, 500
    left = pa.table({"k": rng.integers(0, 3, n1), "t": _values(tp, n1, rng)})
    right = pa.table({"k": rng.integers(0, 3, n2), "t": _values(tp, n2, rng), "rid": np.arange(n2)})
    _check(left, right, ["k"], "t", "left_outer", direction, exact)
    tol = 2.5 if tp in _FLOATS else (datetime.timedelta(seconds=3) if pa.types.is_timestamp(tp) or
                                      pa.types.is_duration(tp) or tp == pa.date64() else 3)
    units = {pa.timestamp("s"): 3, pa.timestamp("ns", "UTC"): 3_000_000_000, pa.duration("ms"): 3000,
             pa.date64(): 3000}.get(tp)
    if tp == pa.date32():
        tol, units = datetime.timedelta(days=3), 3
    _check(left, right, ["k"], "t", "inner", direction, exact, tol, units)


@pytest.mark.parametrize("direction,exact", DIRS)
def test_int64_extremes_with_tolerance(direction, exact):
    lo, hi = -(1 << 63), (1 << 63) - 1
    vals = np.array([lo, lo + 1, lo + 2, -2, -1, 0, 1, 2, hi - 2, hi - 1, hi], np.int64)
    lt, rt = np.repeat(vals, 3), vals[np.random.default_rng(3).permutation(len(vals))]
    left = pa.table({"t": lt})
    right = pa.table({"t": rt, "rid": np.arange(len(rt))})
    for tol in (None, 0, 1, 2, (1 << 62), hi - 1, hi):
        _check(left, right, [], "t", "left_outer", direction, exact, tol)


def test_keys_of_every_kind():
    rng = np.random.default_rng(4)
    n1, n2 = 3000, 2000
    lt, rt = rng.integers(0, 500, n1), rng.integers(0, 500, n2)
    fl = np.array([0.0, -0.0, 1.5, np.nan, -2.0])
    left = pa.table({"f": pa.array(fl[rng.integers(0, 5, n1)], mask=rng.random(n1) < 0.05),
                     "s": pa.array(np.array(["a", "b", "c", "dd"])[rng.integers(0, 4, n1)]),
                     "i": pa.array(rng.integers(0, 4, n1), pa.int32()), "t": lt})
    right = pa.table({"f": pa.array(fl[rng.integers(0, 5, n2)]),
                      "s": pa.array(np.array(["dd", "zz", "b", "a"])[rng.integers(0, 4, n2)]),
                      "i": pa.array(rng.integers(0, 4, n2), pa.int32(), mask=rng.random(n2) < 0.05), "t": rt,
                      "rid": np.arange(n2)})
    for on in (["f"], ["s"], ["i"], ["s", "i"], ["f", "s", "i"]):
        rest = [c for c in ("f", "s", "i") if c not in on]
        for direction, exact in DIRS:
            _check(left.drop(rest), right.drop(rest), on, "t", "left_outer", direction, exact)


def test_weak_hash_is_verified(monkeypatch):
    """With a 2-bit surrogate hash every run head collides with others: only verified heads may match."""
    strong = K.row_hash64
    monkeypatch.setattr(K, "row_hash64", lambda keys, valid=None: strong(keys, valid) & 3)
    rng = np.random.default_rng(5)
    n1, n2 = 5000, 4000
    left = pa.table({"a": rng.integers(0, 20, n1), "b": rng.integers(0, 20, n1), "t": rng.integers(0, 99, n1)})
    right = pa.table({"a": rng.integers(0, 18, n2), "b": rng.integers(0, 20, n2), "t": rng.integers(0, 99, n2),
                      "rid": np.arange(n2)})
    for direction, exact in DIRS:
        _check(left, right, ["a", "b"], "t", "left_outer", direction, exact)
        _check(left, right, ["a", "b"], "t", "inner", direction, exact, tol=4)


def test_nullable_and_string_right_columns():
    rng = np.random.default_rng(6)
    n1, n2 = 4000, 3000
    left = pa.table({"k": rng.integers(0, 50, n1), "t": rng.integers(0, 1000, n1),
                     "name": pa.array(np.array(["x", "y"])[rng.integers(0, 2, n1)])})
    right = pa.table({"k": rng.integers(0, 50, n2), "t": pa.array(rng.integers(0, 1000, n2), mask=rng.random(n2) < .1),
                      "rid": np.arange(n2),
                      "q": pa.array(rng.standard_normal(n2), mask=rng.random(n2) < 0.2),
                      "s": pa.array(np.array(["p", "q", "r"])[rng.integers(0, 3, n2)], mask=rng.random(n2) < 0.2),
                      "b": pa.array(rng.random(n2) < 0.5, mask=rng.random(n2) < 0.2),
                      "h": pa.array(rng.integers(0, 9, n2), pa.int16())})
    for how in ("inner", "left_outer"):
        for direction, exact in DIRS:
            _check(left, right, ["k"], "t", how, direction, exact)


def _trades_quotes(n1: int, n2: int, seed: int):
    rng = np.random.default_rng(seed)
    base = pd.Timestamp("2026-01-02 09:30")
    quotes = pd.DataFrame({"t": base + pd.to_timedelta(np.sort(rng.integers(0, 10**9, n2)), unit="us"),
                           "sym": np.array(["AA", "BB", "CC", "DD"])[rng.integers(0, 4, n2)],
                           "bid": rng.standard_normal(n2), "ask": rng.standard_normal(n2)})
    trades = pd.DataFrame({"t": base + pd.to_timedelta(np.sort(rng.integers(0, 10**9, n1)), unit="us"),
                           "sym": np.array(["AA", "BB", "CC", "EE"])[rng.integers(0, 4, n1)],
                           "price": rng.standard_normal(n1), "qty": rng.integers(1, 100, n1)})
    return trades, quotes


def _same_frame(a: pd.DataFrame, b: pd.DataFrame):
    assert list(a.columns) == list(b.columns)
    for c in a.columns:
        x, y = a[c], b[c]
        if pd.api.types.is_datetime64_any_dtype(x):
            assert (x.astype("datetime64[ns]").astype("int64") == y.astype("datetime64[ns]").astype("int64")).all(), c
        else:
            assert x.isna().tolist() == y.isna().tolist(), c
            assert (x[~x.isna()].astype(str) == y[~y.isna()].astype(str)).all(), c


@pytest.mark.parametrize("direction,exact", DIRS)
@pytest.mark.parametrize("tol", [None, pd.Timedelta(milliseconds=50)])
def test_merge_asof_through_the_api(direction, exact, tol):
    trades, quotes = _trades_quotes(20_000, 30_000, 7)
    exp = pd.merge_asof(trades, quotes, on="t", by="sym", direction=direction, allow_exact_matches=exact,
                        tolerance=tol)
    got = fa.asof_join(trades, quotes, on=["sym"], asof="t", how="left_outer", direction=direction,
                       allow_exact_matches=exact, tolerance=None if tol is None else tol.to_pytimedelta(),
                       engine=_engine(), as_fugue=True).as_pandas()
    _same_frame(got, exp[list(got.columns)])


def test_merge_asof_through_sql():
    trades, quotes = _trades_quotes(20_000, 30_000, 8)
    exp = pd.merge_asof(trades, quotes, on="t", by="sym")
    got = fa.raw_sql("SELECT * FROM", trades, "ASOF LEFT JOIN", quotes,
                     "ON trades.sym = quotes.sym AND trades.t >= quotes.t", engine=_engine(), as_fugue=True).as_pandas()
    _same_frame(got, exp[list(got.columns)])
    got = fa.raw_sql("SELECT * FROM", trades, "AS a ASOF JOIN", quotes, "AS b ON b.sym = a.sym AND b.t > a.t",
                     engine=_engine(), as_fugue=True).as_pandas()
    exp = pd.merge_asof(trades, quotes, on="t", by="sym", direction="forward", allow_exact_matches=False)
    _same_frame(got, exp.dropna(subset=["bid"]).reset_index(drop=True)[list(got.columns)])


@pytest.mark.parametrize("n", [1, 1000, 2_000_001])
def test_search_kernel_against_searchsorted(n):
    """``fb_asof_search`` alone, one run of sorted codes: backward is ``searchsorted(side)`` - 1, forward is
    ``searchsorted(other side)``."""
    rng = np.random.default_rng(n)
    codes = np.sort(rng.integers(0, 1 << 62, n // 2 + 1).astype(np.uint64) * np.uint64(2))
    codes[-1] = np.uint64((1 << 64) - 2)  # above 2^63
    x = np.concatenate([codes[rng.integers(0, len(codes), n)], rng.integers(0, 1 << 63, n).astype(np.uint64)])
    m = len(codes)
    perm = rng.permutation(m).astype(np.int64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    run, off = t(np.zeros(len(x), np.int64)), t(np.array([0, m], np.int64))
    for direction, exact in DIRS:
        got = K.asof_search(run, off, t(x.view(np.int64)), None, t(codes.view(np.int64)), t(perm), K.RANGE_KEY_U64,
                            A.DIRECTIONS.index(direction), exact, None).cpu().numpy()
        b = np.searchsorted(codes, x, "right" if exact else "left") - 1
        f = np.searchsorted(codes, x, "left" if exact else "right")
        if direction == "backward":
            pos = b
        elif direction == "forward":
            pos = np.where(f < m, f, -1)
        else:
            db = x - codes[np.clip(b, 0, m - 1)]
            df = codes[np.clip(f, 0, m - 1)] - x
            pos = np.where(b < 0, np.where(f < m, f, -1), np.where((f >= m) | (db <= df), b, f))
        exp = np.where(pos >= 0, perm[np.clip(pos, 0, m - 1)], -1)
        assert np.array_equal(got, exp), (direction, exact)
