"""EWM_MEAN, EWM_VAR and EWM_STD without a GPU: the builders and ``over()`` rules, every rejection, the SQL spellings
and print -> parse as a fixed point, the exact reference (oracle/ewm.py) against pandas' ``ewm``, and a float64 model of
the ``EwSt`` combine of ``fb_segmented_ewm`` against that reference on random splits into runs, within the bound of
DESIGN §7s.

pandas 3.0.2 differs from the weight definition in three places, which the comparisons leave out on purpose:
  - with ``adjust=False`` and alpha exactly 0.5 (com = 1) its mean after a NULL gap is 2.5 for [1, NaN, 3], not 2.333…
    (it gives the new value the weight 1 - decay); a time decay has com = 1, so this holds for every time gap there;
  - its unbiased variance of a single observation after NULL rows is sometimes 0.0 instead of NaN (rounding of its
    repeated products);
  - it replaces +-inf by NaN before the recurrence; the engine keeps them as observations (the mean stays +-inf, or NaN
    with both signs, and the variance is NaN), as its other aggregates do.
"""
import datetime
import decimal
import math

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from fugue_b200.colmap import ColumnMap
from fugue_b200.column import (AGGREGATES, EWM_HEADS, SCALARS, Kind, col, ewm_alpha, functions as f, is_explicit)
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from oracle.ewm import ewm, ewm_sums, pandas_alpha

import _ewm_model as M

U = 2.0 ** -53


def _item(text: str):
    st = _parse_select(text, "FROM t", "SELECT " + text + " FROM t")
    assert len(st.columns) == 1
    return st.columns[0]


def _same(a, b) -> bool:
    return a.fingerprint() == b.fingerprint()


# ---- builders, over() and SQL --------------------------------------------------------------------------------------
def test_heads_are_window_only():
    for h in EWM_HEADS:
        assert h not in AGGREGATES and h not in SCALARS


def test_builders_and_types():
    sch = Schema("v:float,k:long,t:long")
    for e in (f.ewm_mean("v", alpha=0.1), f.ewm_var(col("v"), com=2), f.ewm_std("v", span=5, bias=True)):
        assert e.kind == Kind.WINDOW and e.infer_type(sch) == pa.float64()
        assert e.infer_alias().output_name == "v"
    assert f.ewm_mean("v", alpha=0.1).kwargs == {"alpha": 0.1, "adjust": True, "ignore_na": False, "min_periods": 0,
                                                 "times": False}
    assert f.ewm_var("v", com=1, adjust=False).kwargs["bias"] is False
    # a bare node runs in a ColumnMap
    ColumnMap("k", f.ewm_mean(col("v"), alpha=0.5).alias("a"), f.ewm_std(col("v"), halflife=3.0).alias("b"))


_RANDOM_ALPHAS = [float(x) for x in np.random.default_rng(9).random(300)] + [0.4392914635525388]


@pytest.mark.parametrize("kw", [dict(com=0.0), dict(com=3.5), dict(span=1), dict(span=7.5), dict(halflife=0.25),
                                dict(halflife=40), dict(alpha=1e-6), dict(alpha=0.5), dict(alpha=1)] +
                         [dict(alpha=a) for a in _RANDOM_ALPHAS if a > 0])
def test_alpha_is_pandas_alpha(kw):
    from pandas.core.window.ewm import get_center_of_mass

    a = ewm_alpha(f.ewm_mean("v", **kw).kwargs)
    com = get_center_of_mass(kw.get("com"), kw.get("span"), kw.get("halflife"), kw.get("alpha"))
    assert a == 1.0 / (1.0 + com) == pandas_alpha(**kw)
    s = pd.Series([1.0, 5.0])
    assert s.ewm(**kw).mean().iloc[1] == pytest.approx((1.0 * (1 - a) + 5.0) / (2 - a), rel=1e-15)


@pytest.mark.parametrize("make", [
    lambda: f.ewm_mean("v"),
    lambda: f.ewm_mean("v", alpha=0.5, com=1),
    lambda: f.ewm_mean("v", alpha=0.0),
    lambda: f.ewm_mean("v", alpha=1.5),
    lambda: f.ewm_mean("v", alpha=True),
    lambda: f.ewm_mean("v", alpha=math.nan),
    lambda: f.ewm_mean("v", com=-0.5),
    lambda: f.ewm_mean("v", span=0.5),
    lambda: f.ewm_mean("v", halflife=0),
    lambda: f.ewm_mean("v", alpha=0.5, adjust=1),
    lambda: f.ewm_mean("v", alpha=0.5, min_periods=-1),
    lambda: f.ewm_mean("v", alpha=0.5, min_periods=1.5),
    lambda: f.ewm_mean("v", alpha=0.5, times=True),
    lambda: f.ewm_mean("v", halflife=datetime.timedelta(days=1)),
    lambda: f.ewm_mean("v", halflife=datetime.timedelta(0), times=True),
    lambda: f.ewm_mean("*", alpha=0.5),
    lambda: f.ewm_mean(f.sum(col("v")), alpha=0.5),
    lambda: f.ewm_mean("v", alpha=0.5).over(running=True),
    lambda: f.ewm_mean("v", alpha=0.5).over(rows=(-2, 0), partition_by=["k"], order_by=["t"]),
    lambda: f.ewm_var("v", alpha=0.5).over(range=(-2, 0), partition_by=["k"], order_by=["t"]),
    lambda: f.ewm_std("v", alpha=0.5).over(running=True, partition_by=["k"], order_by=["t"]),
    lambda: f.ewm_mean("v", halflife=2, times=True).over(partition_by=["k"], order_by=[("t", False)]),
    lambda: f.ewm_mean("v", halflife=2, times=True).over(partition_by=["k"], order_by=["t", "k"]),
    lambda: f.ewm_mean("v", halflife=2, times=True).over(partition_by=["k"]),
])
def test_rejections(make):
    with pytest.raises(ValueError):
        make()


@pytest.mark.parametrize("make", [
    lambda: f.ewm_mean("v", halflife=2, times=True, ignore_na=True),
    lambda: f.ewm_var("v", halflife=2, times=True),
    lambda: f.ewm_std("v", halflife=datetime.timedelta(hours=1), times=True),
])
def test_not_implemented(make):
    with pytest.raises(NotImplementedError):
        make()


def test_explicit_node():
    e = f.ewm_std("v", alpha=0.25, bias=True).over(partition_by=["k"], order_by=["t"])
    assert is_explicit(e) and e.kwargs["bias"] is True and "running" not in e.kwargs
    e = f.ewm_mean("v", halflife=datetime.timedelta(hours=6), times=True).over(partition_by=["k"], order_by=["t"])
    assert e.kwargs["halflife"] == datetime.timedelta(hours=6)


@pytest.mark.parametrize("text, node", [
    ("EWM_MEAN(v, 0.1) OVER (PARTITION BY k ORDER BY t)",
     lambda: f.ewm_mean("v", alpha=0.1).over(partition_by=["k"], order_by=["t"])),
    ("EWM_VAR(v, 0.25, FALSE) OVER (ORDER BY t)",
     lambda: f.ewm_var("v", alpha=0.25, adjust=False).over(order_by=["t"])),
    ("EWM_STD(v, 1) OVER (PARTITION BY k ORDER BY t DESC)",
     lambda: f.ewm_std("v", alpha=1.0).over(partition_by=["k"], order_by=[("t", False)])),
    ("ewm_mean(v, INTERVAL '2' DAY, TRUE) OVER (PARTITION BY k ORDER BY t)",
     lambda: f.ewm_mean("v", halflife=datetime.timedelta(days=2), times=True).over(partition_by=["k"], order_by=["t"])),
    ("EWM_MEAN(v, INTERVAL '0 06:00:00' DAY TO SECOND) OVER (ORDER BY t)",
     lambda: f.ewm_mean("v", halflife=datetime.timedelta(hours=6), times=True).over(order_by=["t"])),
])
def test_sql_spellings_and_round_trip(text, node):
    e = _item(text)
    assert _same(e.alias(""), node())
    again = _item(str(e))
    assert _same(again, e)
    assert str(again) == str(e)


@pytest.mark.parametrize("text, exc", [
    ("EWM_MEAN(v, 0.5) OVER (ORDER BY t ROWS BETWEEN 1 PRECEDING AND CURRENT ROW)", ValueError),
    ("EWM_MEAN(v, 0.5) OVER (ORDER BY t RANGE BETWEEN 1 PRECEDING AND CURRENT ROW)", ValueError),
    ("EWM_MEAN(v, 0) OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v, 1.5) OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v, 'a') OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v, k) OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v, 0.5, 1) OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v) OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v, 0.5, TRUE, 1) OVER (ORDER BY t)", ValueError),
    ("EWM_MEAN(v, INTERVAL '1' DAY) OVER (ORDER BY t DESC)", ValueError),
    ("EWM_MEAN(v, INTERVAL '1' DAY) OVER (ORDER BY t, k)", ValueError),
    ("EWM_VAR(v, INTERVAL '1' DAY) OVER (ORDER BY t)", NotImplementedError),
    ("EWM_MEAN(v, 0.5)", NotImplementedError),
])
def test_sql_rejections(text, exc):
    with pytest.raises(exc):
        _item(text)


def test_non_sql_options_print():
    e = f.ewm_var("v", com=2, adjust=False, ignore_na=True, min_periods=3, bias=True).over(order_by=["t"])
    assert str(e) == "EWM_VAR(v,com=2.0,adjust=FALSE,ignore_na=TRUE,min_periods=3,bias=TRUE) OVER (ORDER BY t)"


# ---- the reference against pandas ----------------------------------------------------------------------------------
def _pandas_quirk(vals, a, adjust):
    return not adjust and a == 0.5 and any(x is None for x in vals)


def _check_against_pandas(vals, kw, adjust, ignore_na, min_periods=0):
    a = pandas_alpha(**kw)
    s = pd.Series([np.nan if x is None else x for x in vals], dtype=float)
    e = s.ewm(adjust=adjust, ignore_na=ignore_na, min_periods=min_periods, **kw)
    for fn, bias, got in (("EWM_MEAN", False, e.mean()), ("EWM_VAR", False, e.var()), ("EWM_VAR", True, e.var(bias=True)),
                          ("EWM_STD", False, e.std()), ("EWM_STD", True, e.std(bias=True))):
        if fn == "EWM_MEAN" and _pandas_quirk(vals, a, adjust):
            continue
        ref = ewm(fn, vals, a, adjust, ignore_na, bias, min_periods)
        for i, (r, p) in enumerate(zip(ref, got)):
            if r is None:
                # pandas' unbiased variance of one observation after NULL rows is sometimes 0.0
                assert math.isnan(p) or (not bias and fn != "EWM_MEAN" and p == 0.0), (fn, i, vals, kw)
            else:
                assert p == pytest.approx(r, rel=1e-11, abs=1e-13), (fn, bias, i, vals, kw, adjust, ignore_na)


@pytest.mark.parametrize("seed", range(40))
def test_reference_against_pandas(seed):
    rng = np.random.default_rng(seed)
    decays = [dict(alpha=0.1), dict(alpha=0.5), dict(alpha=0.9), dict(alpha=1.0), dict(com=0.0), dict(com=2.5),
              dict(span=1), dict(span=6.5), dict(halflife=0.7), dict(halflife=12)]
    for _ in range(5):
        n = int(rng.integers(0, 4)) if rng.random() < 0.4 else int(rng.integers(4, 40))
        lead = int(rng.integers(0, 3))
        vals = [None] * min(lead, n) + [None if rng.random() < 0.2 else float(rng.normal(3, 2)) for _ in range(n - lead)]
        kw = decays[int(rng.integers(len(decays)))]
        _check_against_pandas(vals, kw, bool(rng.integers(2)), bool(rng.integers(2)), int(rng.integers(0, 4)))


def test_reference_against_pandas_groupby():
    rng = np.random.default_rng(7)
    k = rng.integers(0, 6, 300)
    v = np.where(rng.random(300) < 0.15, np.nan, rng.normal(size=300))
    df = pd.DataFrame({"k": k, "v": v})
    got = df.groupby("k")["v"].ewm(alpha=0.3, adjust=False).mean().reset_index(level=0, drop=True).sort_index()
    for key in range(6):
        idx = np.flatnonzero(k == key)
        ref = ewm("EWM_MEAN", [None if np.isnan(x) else float(x) for x in v[idx]], 0.3, adjust=False)
        for i, r in zip(idx, ref):
            assert (r is None and np.isnan(got[i])) or got[i] == pytest.approx(r, rel=1e-12)


def test_reference_times_against_pandas():
    rng = np.random.default_rng(3)
    t = np.cumsum(rng.integers(0, 5, 60)) * 3_600_000_000  # microseconds, ties included
    v = [None if rng.random() < 0.2 else float(x) for x in rng.normal(size=60)]
    times = pd.to_datetime(t, unit="us")
    # a time decay runs with com = 1, so without adjust pandas takes its alpha = 0.5 branch (new weight 1 - decay)
    for adjust in (True,):
        got = pd.Series([np.nan if x is None else x for x in v]).ewm(
            halflife=pd.Timedelta(hours=5), times=times, adjust=adjust).mean()
        ref = ewm("EWM_MEAN", v, 0.5, adjust, times=[int(x) for x in t], halflife=5 * 3_600_000_000)
        for r, p in zip(ref, got):
            assert (r is None and np.isnan(p)) or p == pytest.approx(r, rel=1e-12)


def test_pandas_quirks_are_what_the_tests_skip():
    s = pd.Series([1.0, np.nan, 3.0])
    assert s.ewm(alpha=0.5, adjust=False).mean().iloc[2] == 2.5
    assert ewm("EWM_MEAN", [1.0, None, 3.0], 0.5, adjust=False)[2] == pytest.approx(7 / 3)
    assert s.ewm(alpha=0.4, adjust=False).mean().iloc[2] == pytest.approx(
        ewm("EWM_MEAN", [1.0, None, 3.0], 0.4, adjust=False)[2], rel=1e-15)
    assert pd.Series([1.0, np.inf]).ewm(alpha=0.3).mean().iloc[1] == 1.0  # pandas drops the inf
    assert ewm("EWM_MEAN", [1.0, math.inf], 0.3)[1] == math.inf


def test_edge_values():
    assert ewm("EWM_VAR", [2.0, 2.0, None, 2.0], 0.3) == [None, 0.0, 0.0, 0.0]
    m = ewm("EWM_MEAN", [1.0, math.inf, 2.0, -math.inf], 0.3)
    assert m[1:3] == [math.inf, math.inf] and math.isnan(m[3])
    assert math.isnan(ewm("EWM_VAR", [1.0, math.inf, 2.0], 0.3, bias=True)[2])
    assert ewm("EWM_MEAN", [None, None, 4.0, math.nan, None], 0.3) == [None, None, 4.0, 4.0, 4.0]
    assert ewm("EWM_MEAN", [1.0, 2.0, 3.0], 0.3, min_periods=2)[:2] == [None, pytest.approx((0.7 + 2.0) / 1.7)]


# ---- the float64 model of the combine ------------------------------------------------------------------------------
def _bound_ok(fn, got, ref, spread, depth):
    """DESIGN §7s: |error| <= 4 (D + 8) u (|ref| + spread) for a result D combines deep; for the mean, spread = max
    |x - mean| over the observations, for C it is W max |x - mean| (max |x - mean| + |mean|), for W and W2 0."""
    return abs(got - ref) <= 4 * (depth + 8) * U * (abs(ref) + spread)


def _exact(vals, alpha, adjust, ignore_na, times=None, halflife=None, decimal=False):
    return ewm_sums(vals, alpha, adjust, ignore_na, times, halflife, decimal)


def _check_model(got, ex, vals, adjust, depth, check_c=True):
    """Each row of the model (count, mean, W, W2, C) against the exact sums, within the bound.  Without adjust the
    state keeps weight shares, so W is 1 and W2, C are the exact W2 / W^2 and C / W."""
    with decimal.localcontext(decimal.Context(prec=60)):  # the decimal sums keep their 60 digits
        _check_model_rows(got, ex, vals, adjust, depth, check_c)


def _check_model_rows(got, ex, vals, adjust, depth, check_c):
    lo, hi = math.inf, -math.inf
    for i, (g, e) in enumerate(zip(got, ex)):
        x = vals[i]
        if x is not None and x == x:
            lo, hi = min(lo, x), max(hi, x)
        if e is None:
            assert g[0] == 0
            continue
        c, W, W2, S1, S2, _ = e
        assert g[0] == c
        mean = S1 / W
        C = S2 - S1 * mean
        if not adjust:
            W, W2, C = W / W, W2 / (W * W), C / W
        m = float(mean)
        spread = max(hi - m, m - lo)
        assert _bound_ok("mean", g[1], m, spread, depth), (i, g, m)
        assert _bound_ok("W", g[2], float(W), 0.0, depth) and _bound_ok("W2", g[3], float(W2), 0.0, depth), (i, g)
        if check_c:
            assert _bound_ok("C", g[4], float(C), float(W) * spread * (spread + abs(m)), depth), (i, g[4], float(C))


@pytest.mark.parametrize("seed", range(30))
def test_model_combine_on_random_splits(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 120))
    vals = [None if rng.random() < 0.2 else (float(rng.normal(50, 10)) if rng.random() < 0.97 else math.nan)
            for _ in range(n)]
    alpha = [0.05, 0.3, 0.5, 0.85, 1.0][seed % 5]
    adjust, ignore_na = bool(seed & 1), bool(seed & 2)
    timed = seed % 7 == 3
    if timed:
        ts = list(np.cumsum(rng.integers(0, 4, n)))
        op, ignore_na = M.make_op(0.5, adjust, False, 1 / 2.5), False
        ex = _exact(vals, 0.5, adjust, False, ts, 2.5)
    else:
        ts = list(range(n))
        op = M.make_op(alpha, adjust, ignore_na)
        ex = _exact(vals, alpha, adjust, ignore_na)
    cuts = sorted(rng.choice(np.arange(1, n + 1), size=min(n, int(rng.integers(0, 12))), replace=False).tolist())
    got = M.fold(op, vals, [int(x) for x in ts], cuts)
    _check_model(got, ex, vals, adjust, n, check_c=not timed)  # C of a time decay has no head to read it


def _long_gapped(n):
    """n rows, every other one NULL: without adjust pandas' total T shrinks by beta + alpha at every gap"""
    rng = np.random.default_rng(41)
    return [None if i % 2 else float(rng.normal(1, 0.1)) for i in range(n)]


def test_model_long_partition_with_gaps_without_adjust():
    n = 100_000
    vals = _long_gapped(n)
    op = M.make_op(0.3, False, False)
    got = M.fold(op, vals, list(range(n)), list(range(2048, n, 2048)))
    ex = _exact(vals, 0.3, False, False, decimal=True)
    _check_model(got, ex, vals, False, 2048 + n // 2048)
    # the last rows against pandas, which runs the same recurrence sequentially
    s = pd.Series([np.nan if x is None else x for x in vals]).ewm(alpha=0.3, adjust=False)
    for i in (7000, n - 2, n - 1):
        assert got[i][1] == pytest.approx(s.mean().iloc[i], rel=1e-12)


def test_model_long_time_decay_without_adjust():
    n = 100_000
    rng = np.random.default_rng(42)
    ts = [int(x) for x in np.cumsum(rng.integers(0, 3, n))]  # ties, steps much shorter than the halflife
    vals = [None if rng.random() < 0.05 else float(rng.normal(3, 1)) for _ in range(n)]
    for adjust in (False, True):
        got = M.fold(M.make_op(0.5, adjust, False, 1 / 60), vals, ts, list(range(2048, n, 2048)))
        ex = _exact(vals, 0.5, adjust, False, ts, 60)
        _check_model(got, ex, vals, adjust, 2048 + n // 2048, check_c=False)


def test_model_constant_runs_are_exactly_zero():
    op = M.make_op(0.3, False, False)
    vals = [7.25] * 40 + [None] * 3 + [7.25] * 10
    for cuts in ([], [5, 17, 41], list(range(1, 53, 2))):
        for g in M.fold(op, vals, list(range(len(vals))), cuts):
            assert g[1] == 7.25 and g[4] == 0.0


def test_model_infinities():
    op = M.make_op(0.3, True, False)
    got = M.fold(op, [1.0, math.inf, 2.0, -math.inf, 3.0], list(range(5)), [2, 3])
    assert got[1][1] == math.inf and got[2][1] == math.inf and math.isnan(got[3][1]) and math.isnan(got[1][4])


def test_shifted_data_chan_holds_textbook_fails():
    rng = np.random.default_rng(5)
    n = 400
    vals = [float(x) for x in 1e9 + 1e-3 * rng.standard_normal(n)]
    op = M.make_op(0.1, True, False)
    ex = _exact(vals, 0.1, True, False)
    got = M.fold(op, vals, list(range(n)), [37, 100, 101, 256])
    beta, W, S1, S2 = 0.9, 0.0, 0.0, 0.0
    textbook_fails = 0
    for i, (g, e) in enumerate(zip(got, ex)):
        c, We, W2e, S1e, S2e, _ = e
        mean = S1e / We
        C = float(S2e - S1e * mean)
        spread = max(abs(x - float(mean)) for x in vals[:i + 1])
        cs = float(We) * spread * (spread + abs(float(mean)))
        assert _bound_ok("C", g[4], C, cs, n)
        W, S1, S2 = W * beta + 1.0, S1 * beta + vals[i], S2 * beta + vals[i] * vals[i]
        textbook = S2 - S1 * S1 / W
        textbook_fails += not _bound_ok("C", textbook, C, cs, n)
    assert textbook_fails > n // 2
