"""Range joins on the H100 (DESIGN §7r): ``fa.range_join`` against ``oracle.range_join`` row by row in output order,
at edge sizes, on one run of 10^6 intervals, at 10^7 left rows x 10^6 intervals, on every value type with NULLs /
NaN / -0.0 / infinities / uint64 >= 2^63 / the int64 extremes as bounds, on zero-width, reversed and touching
intervals under each ``closed``, on integer / float / string / two-column keys (a weak surrogate hash included),
with a left row of more than 10^5 matches and with one interval nesting 10^5 others; and against ``pandas.merge``
followed by a filter through ``fa.range_join`` and ``fa.raw_sql``."""
from typing import Any, List

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from oracle import range_join as R

_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _device(left: pa.Table, right: pa.Table, on, at="t", start="s", end="e", **kw) -> pa.Table:
    return fa.range_join(left, right, on=on, at=at, start=start, end=end, engine=_engine(), as_fugue=True,
                         **kw).as_arrow()


def _same_floats(a, b) -> bool:
    return len(a) == len(b) and all(x == y or (x != x and y != y) for x, y in zip(a, b))


def _check(left: pa.Table, right: pa.Table, on, how="inner", closed="both", at="t", start="s", end="e"):
    """The device against the oracle, column by column in output order."""
    got = _device(left, right, on, at, start, end, how=how, closed=closed)
    exp = R.range_join(left, right, on, at, start, end, how, closed)
    assert got.column_names == exp.column_names
    for n in exp.column_names:
        a, b = _plain(got.column(n)), _plain(exp.column(n))
        assert a == b or _same_floats(a, b), (n, how, closed)
    return got


def _plain(c: Any) -> list:
    """A column as Python values; timestamps as their storage integers (a zoned timestamp's Python value costs a
    time-zone lookup per row)."""
    return (c.cast(pa.int64()) if pa.types.is_timestamp(c.type) else c).to_pylist()


def _np_pairs(lk, lt, rk, rs, re_, closed="both", how="inner", lok=None, rok=None):
    n1, n2 = len(lk), len(rk)
    return R.match_pairs_np(lk, R.codes_np(lt), np.ones(n1, bool) if lok is None else lok, rk, R.codes_np(rs),
                            R.codes_np(re_), np.ones(n2, bool) if rok is None else rok, closed, how)


def _check_np(got: pa.Table, li: np.ndarray, ri: np.ndarray, lcol: str = "i"):
    assert got.num_rows == len(li)
    assert np.array_equal(got.column(lcol).to_numpy(), li)
    assert np.array_equal(got.column("rid").fill_null(-1).to_numpy(), ri)


@pytest.mark.parametrize("n1,n2", [(0, 0), (0, 5), (5, 0), (1, 1), (1, 3), (3, 1), (2047, 2049), (2049, 2047),
                                   (4095, 4097), (4097, 1)])
@pytest.mark.parametrize("closed", R.CLOSED)
def test_edge_sizes(n1, n2, closed):
    rng = np.random.default_rng(n1 * 7 + n2 + len(closed))
    s = rng.integers(0, 300, n2)
    left = pa.table({"k": rng.integers(0, 9, n1), "t": rng.integers(-5, 320, n1), "v": rng.standard_normal(n1)})
    right = pa.table({"k": rng.integers(0, 8, n2), "s": s, "e": s + rng.integers(-2, 30, n2), "rid": np.arange(n2)})
    for how in R.HOWS:
        _check(left, right, ["k"], how, closed)
    _check(left, right.drop(["k"]), [], "inner", closed)


def test_one_long_run():
    """One key whose run holds 10^6 intervals."""
    rng = np.random.default_rng(1)
    n1, n2 = 300_000, 1_000_000
    lt, rs = rng.integers(-10, 3_000_010, n1), rng.integers(0, 3_000_000, n2)
    re_ = rs + rng.integers(0, 20, n2)
    left = pa.table({"k": np.full(n1, 5), "t": lt, "i": np.arange(n1)})
    right = pa.table({"k": np.full(n2, 5), "s": rs, "e": re_, "rid": np.arange(n2)})
    for closed in R.CLOSED:
        got = _device(left, right, ["k"], how="left_outer", closed=closed)
        _check_np(got, *_np_pairs(np.full(n1, 5), lt, np.full(n2, 5), rs, re_, closed, "left_outer"))


@pytest.mark.parametrize("how", R.HOWS)
def test_ten_million_left_rows(how):
    """10^7 left rows x 10^6 intervals with 65 536 keys, timestamps."""
    rng = np.random.default_rng(2)
    n1, n2, nk = 10_000_000, 1_000_000, 65_536
    lk, rk = rng.integers(0, nk + 100, n1), rng.integers(0, nk, n2)
    lt, rs = rng.integers(0, 1 << 30, n1), rng.integers(0, 1 << 30, n2)
    re_ = rs + rng.integers(0, 1 << 27, n2)  # about one interval in force at a time per key
    left = pa.table({"k": lk, "t": pa.array(lt, pa.timestamp("us")), "i": np.arange(n1)})
    right = pa.table({"k": rk, "s": pa.array(rs, pa.timestamp("us")), "e": pa.array(re_, pa.timestamp("us")),
                      "rid": np.arange(n2)})
    got = _device(left, right, ["k"], how=how)
    li, ri = _np_pairs(lk, lt, rk, rs, re_, "both", how)
    assert len(li) > n1 // 4
    _check_np(got, li, ri)
    assert np.array_equal(got.column("k").to_numpy(), lk[li])


_INTS = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64()]
_TEMPORAL = [pa.date32(), pa.date64(), pa.timestamp("s"), pa.timestamp("ns", "UTC"), pa.duration("ms"),
             pa.time64("us")]
_FLOATS = [pa.float16(), pa.float32(), pa.float64()]


def _values(tp: pa.DataType, n: int, rng: np.random.Generator) -> pa.Array:
    """n values of ``tp`` with NULLs, few distinct values (ties, touching and zero-width intervals), and the type's
    edge values."""
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
        v[rng.random(n) < 0.05] = np.uint64(0)
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
def test_every_value_type(tp):
    rng = np.random.default_rng(len(str(tp)) * 31)
    n1, n2 = 700, 400
    left = pa.table({"k": rng.integers(0, 3, n1), "t": _values(tp, n1, rng)})
    right = pa.table({"k": rng.integers(0, 3, n2), "s": _values(tp, n2, rng), "e": _values(tp, n2, rng),
                      "rid": np.arange(n2)})
    for closed in R.CLOSED:
        for how in R.HOWS:
            _check(left, right, ["k"], how, closed)
    one = pa.table({"p": _values(tp, n2, rng), "rid": np.arange(n2)})  # start and end one column: points
    _check(left, one, [], "left_outer", "both", start="p", end="p")


def test_int64_extremes_as_bounds():
    lo, hi = -(1 << 63), (1 << 63) - 1
    vals = np.array([lo, lo + 1, -1, 0, 1, hi - 1, hi], np.int64)
    s = np.array([lo, lo, lo + 1, 0, hi, hi - 1, -1, 1], np.int64)
    e = np.array([hi, lo, 0, 0, hi, hi, lo, 1], np.int64)
    left = pa.table({"t": np.repeat(vals, 2)})
    right = pa.table({"s": s, "e": e, "rid": np.arange(len(s))})
    for closed in R.CLOSED:
        for how in R.HOWS:
            _check(left, right, [], how, closed)


@pytest.mark.parametrize("closed", R.CLOSED)
def test_zero_width_reversed_and_touching(closed):
    left = pa.table({"t": [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10]})
    right = pa.table({"s": [2, 2, 3, 5, 5, 7, 9, 8, 4], "e": [2, 3, 5, 5, 7, 9, 9, 7, 4], "rid": range(9)})
    _check(left, right, [], "left_outer", closed)
    _check(left, right, [], "inner", closed)


def test_keys_of_every_kind():
    rng = np.random.default_rng(4)
    n1, n2 = 3000, 2000
    lt, rs = rng.integers(0, 500, n1), rng.integers(0, 500, n2)
    fl = np.array([0.0, -0.0, 1.5, np.nan, -2.0])
    left = pa.table({"f": pa.array(fl[rng.integers(0, 5, n1)], mask=rng.random(n1) < 0.05),
                     "g": pa.array(np.array(["a", "b", "c", "dd"])[rng.integers(0, 4, n1)]),
                     "i": pa.array(rng.integers(0, 4, n1), pa.int32()), "t": lt})
    right = pa.table({"f": pa.array(fl[rng.integers(0, 5, n2)]),
                      "g": pa.array(np.array(["dd", "zz", "b", "a"])[rng.integers(0, 4, n2)]),
                      "i": pa.array(rng.integers(0, 4, n2), pa.int32(), mask=rng.random(n2) < 0.05), "s": rs,
                      "e": rs + rng.integers(0, 40, n2), "rid": np.arange(n2)})
    for on in (["f"], ["g"], ["i"], ["g", "i"], ["f", "g", "i"]):
        rest = [c for c in ("f", "g", "i") if c not in on]
        for closed in R.CLOSED:
            _check(left.drop(rest), right.drop(rest), on, "left_outer", closed)


def test_weak_hash_is_verified(monkeypatch):
    """With a 2-bit surrogate hash every run head collides with others: only verified heads may match."""
    strong = K.row_hash64
    monkeypatch.setattr(K, "row_hash64", lambda keys, valid=None: strong(keys, valid) & 3)
    rng = np.random.default_rng(5)
    n1, n2 = 5000, 4000
    s = rng.integers(0, 99, n2)
    left = pa.table({"a": rng.integers(0, 20, n1), "b": rng.integers(0, 20, n1), "t": rng.integers(0, 99, n1)})
    right = pa.table({"a": rng.integers(0, 18, n2), "b": rng.integers(0, 20, n2), "s": s,
                      "e": s + rng.integers(0, 9, n2), "rid": np.arange(n2)})
    for closed in R.CLOSED:
        _check(left, right, ["a", "b"], "left_outer", closed)
        _check(left, right, ["a", "b"], "inner", closed)


def test_row_with_many_matches():
    """One left row inside 150 000 intervals, its neighbours inside few."""
    rng = np.random.default_rng(10)
    n2 = 200_000
    rs = rng.integers(0, 1_000_000, n2)
    re_ = np.where(np.arange(n2) < 150_000, 2_000_000, rs + 5)
    lt = np.array([1_500_000, 3, 500_000, 999_999, 2_000_001])
    left = pa.table({"t": lt, "i": np.arange(5)})
    right = pa.table({"s": rs, "e": re_, "rid": np.arange(n2)})
    got = _device(left, right, [], how="left_outer")
    li, ri = _np_pairs(np.zeros(5, np.int64), lt, np.zeros(n2, np.int64), rs, re_, "both", "left_outer")
    assert (li == 0).sum() > 100_000
    _check_np(got, li, ri)


def test_adversarial_nesting():
    """One interval spanning the whole run, then 10^5 short ones: every left row meets the long one and at most
    one short one."""
    n = 100_000
    rs = np.r_[0, np.arange(1, n + 1) * 10]
    re_ = np.r_[n * 10 + 100, np.arange(1, n + 1) * 10 + 3]
    rng = np.random.default_rng(11)
    n1 = 1_000_000
    lt = rng.integers(-5, n * 10 + 110, n1)
    left = pa.table({"k": np.zeros(n1, np.int64), "t": lt, "i": np.arange(n1)})
    right = pa.table({"k": np.zeros(n + 1, np.int64), "s": rs, "e": re_, "rid": np.arange(n + 1)})
    for closed in R.CLOSED:
        got = _device(left, right, ["k"], how="left_outer", closed=closed)
        _check_np(got, *_np_pairs(np.zeros(n1, np.int64), lt, np.zeros(n + 1, np.int64), rs, re_, closed,
                                  "left_outer"))


def test_nullable_and_string_right_columns():
    rng = np.random.default_rng(6)
    n1, n2 = 4000, 3000
    s = rng.integers(0, 1000, n2)
    left = pa.table({"k": rng.integers(0, 50, n1), "t": rng.integers(0, 1000, n1),
                     "name": pa.array(np.array(["x", "y"])[rng.integers(0, 2, n1)])})
    right = pa.table({"k": rng.integers(0, 50, n2), "s": pa.array(s, mask=rng.random(n2) < .1),
                      "e": pa.array(s + rng.integers(0, 60, n2), mask=rng.random(n2) < .1), "rid": np.arange(n2),
                      "q": pa.array(rng.standard_normal(n2), mask=rng.random(n2) < 0.2),
                      "g": pa.array(np.array(["p", "q", "r"])[rng.integers(0, 3, n2)], mask=rng.random(n2) < 0.2),
                      "b": pa.array(rng.random(n2) < 0.5, mask=rng.random(n2) < 0.2),
                      "h": pa.array(rng.integers(0, 9, n2), pa.int16())})
    for how in R.HOWS:
        for closed in R.CLOSED:
            _check(left, right, ["k"], how, closed)


def _orders_prices(n1: int, n2: int, seed: int):
    rng = np.random.default_rng(seed)
    base = pd.Timestamp("2026-01-02")
    frm = base + pd.to_timedelta(rng.integers(0, 10**9, n2), unit="s")
    prices = pd.DataFrame({"sku": rng.integers(0, 300, n2), "valid_from": frm,
                           "valid_to": frm + pd.to_timedelta(rng.integers(0, 10**7, n2), unit="s"),
                           "price": rng.standard_normal(n2)})
    orders = pd.DataFrame({"sku": rng.integers(0, 320, n1), "qty": rng.integers(1, 9, n1),
                           "ts": base + pd.to_timedelta(rng.integers(0, 10**9, n1), unit="s")})
    return orders, prices


def _merge_filter(orders, prices, closed, how):
    m = orders.reset_index().merge(prices.reset_index(), on="sku", suffixes=("", "_r"))
    lo = m.valid_from <= m.ts if closed in ("both", "left") else m.valid_from < m.ts
    hi = m.ts <= m.valid_to if closed in ("both", "right") else m.ts < m.valid_to
    m = m[lo & hi].sort_values(["index", "valid_from", "index_r"], kind="stable")
    if how == "left_outer":
        lone = orders.reset_index()[~orders.index.isin(m["index"])]
        m = pd.concat([m, lone]).sort_values(["index", "valid_from", "index_r"], kind="stable", na_position="last")
    return m.drop(columns=["index", "index_r"]).reset_index(drop=True)


def _same_frame(a: pd.DataFrame, b: pd.DataFrame):
    assert list(a.columns) == list(b.columns) and len(a) == len(b)
    for c in a.columns:
        x, y = a[c], b[c]
        assert x.isna().tolist() == y.isna().tolist(), c
        if pd.api.types.is_datetime64_any_dtype(x):
            x, y = x.astype("datetime64[ns]").astype("int64"), y.astype("datetime64[ns]").astype("int64")
        assert (x[~a[c].isna()].astype(str) == y[~b[c].isna()].astype(str)).all(), c


@pytest.mark.parametrize("closed", R.CLOSED)
@pytest.mark.parametrize("how", R.HOWS)
def test_merge_and_filter_through_the_api(closed, how):
    orders, prices = _orders_prices(20_000, 30_000, 7)
    got = fa.range_join(orders, prices, on=["sku"], at="ts", start="valid_from", end="valid_to", how=how,
                        closed=closed, engine=_engine(), as_fugue=True).as_pandas()
    _same_frame(got, _merge_filter(orders, prices, closed, how)[list(got.columns)])


def test_merge_and_filter_through_sql():
    orders, prices = _orders_prices(20_000, 30_000, 8)
    got = fa.raw_sql("SELECT * FROM", orders, "LEFT JOIN", prices,
                     "ON orders.sku = prices.sku AND orders.ts BETWEEN prices.valid_from AND prices.valid_to",
                     engine=_engine(), as_fugue=True).as_pandas()
    _same_frame(got, _merge_filter(orders, prices, "both", "left_outer")[list(got.columns)])
    got = fa.raw_sql("SELECT * FROM", orders, "AS o JOIN", prices,
                     "AS p ON p.sku = o.sku AND p.valid_from <= o.ts AND p.valid_to > o.ts",
                     engine=_engine(), as_fugue=True).as_pandas()
    _same_frame(got, _merge_filter(orders, prices, "left", "inner")[list(got.columns)])
