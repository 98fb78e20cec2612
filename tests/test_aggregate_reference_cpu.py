"""The plain-Python aggregate reference (tests/_aggregate_reference.py) against pandas, numpy and scipy on finite
inputs, and its reading of the edge values of every column type."""
import datetime
import math

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
from scipy import stats

import _aggregate_reference as R
from fugue_b200.column import AGGREGATES
from oracle import groupby as og

RNG = np.random.default_rng(7)
GROUPS = [RNG.standard_normal(n) * 10.0 ** RNG.integers(-3, 4) + RNG.integers(-5, 5) for n in (1, 2, 3, 4, 17, 500)]
GROUPS += [np.array([1.5, 1.5, 1.5, 1.5]), np.array([0.0, -0.0, 0.0, 2.0, -3.0])]


def close(got, want, rel=1e-12, abs_tol=1e-300):
    if want is None or (isinstance(want, float) and math.isnan(want)):
        return got is None or (isinstance(got, float) and math.isnan(got))
    return math.isclose(got, want, rel_tol=rel, abs_tol=abs_tol)


@pytest.mark.parametrize("vals", GROUPS, ids=lambda v: str(len(v)))
def test_basic_and_pick_match_pandas(vals):
    s = pd.Series(vals)
    x = vals.tolist()
    assert R.aggregate("COUNT", pa.float64(), x) == s.count()
    assert close(R.aggregate("SUM", pa.float64(), x), s.sum())
    assert close(R.aggregate("AVG", pa.float64(), x), s.mean())
    assert R.aggregate("MIN", pa.float64(), x) == s.min() and R.aggregate("MAX", pa.float64(), x) == s.max()
    assert R.aggregate("FIRST", pa.float64(), [None] + x) == x[0]
    assert R.aggregate("LAST", pa.float64(), x + [None]) == x[-1]
    ints = np.round(vals * 1000).astype(np.int64)
    assert R.aggregate("SUM", pa.int64(), ints.tolist()) == int(ints.sum())
    assert close(R.aggregate("AVG", pa.int64(), ints.tolist()), float(ints.mean()))


@pytest.mark.parametrize("vals", GROUPS, ids=lambda v: str(len(v)))
def test_variances_and_shapes_match_pandas_and_scipy(vals):
    s = pd.Series(vals)
    x = vals.tolist()
    want = {"VAR_SAMP": s.var(), "VAR_POP": s.var(ddof=0), "STDDEV_SAMP": s.std(), "STDDEV_POP": s.std(ddof=0),
            "SKEWNESS": s.skew(), "KURTOSIS": s.kurt()}
    if len(x) >= 1:
        flat = np.ptp(vals) == 0
        want["SKEWNESS_POP"] = 0.0 if flat else stats.skew(vals, bias=True)
        want["KURTOSIS_POP"] = 0.0 if flat else stats.kurtosis(vals, bias=True)
    if np.ptp(vals) == 0 and len(x) >= 3:  # pandas reports 0 for a constant series; so does the engine
        want["SKEWNESS"] = 0.0
        want["KURTOSIS"] = 0.0 if len(x) >= 4 else None
    for fn, w in want.items():
        w = None if w is None or (isinstance(w, float) and math.isnan(w)) else float(w)
        assert close(R.aggregate(fn, pa.float64(), x), w, rel=1e-9, abs_tol=1e-12), fn


@pytest.mark.parametrize("vals", GROUPS[2:], ids=lambda v: str(len(v)))
def test_pair_functions_match_pandas_and_numpy(vals):
    x = vals.tolist()
    y = (3.0 * vals + RNG.standard_normal(len(vals))).tolist()
    xs, ys = pd.Series(x), pd.Series(y)
    slope, icept = np.polyfit(x, y, 1) if np.ptp(vals) > 0 else (None, None)
    mx, my = np.mean(x), np.mean(y)
    want = {"CORR": xs.corr(ys), "COVAR_SAMP": xs.cov(ys), "COVAR_POP": xs.cov(ys, ddof=0), "REGR_COUNT": len(x),
            "REGR_AVGX": mx, "REGR_AVGY": my, "REGR_SXX": float(((xs - mx) ** 2).sum()),
            "REGR_SYY": float(((ys - my) ** 2).sum()), "REGR_SXY": float(((xs - mx) * (ys - my)).sum()),
            "REGR_SLOPE": slope, "REGR_INTERCEPT": icept, "REGR_R2": xs.corr(ys) ** 2 if np.ptp(vals) > 0 else None}
    for fn, w in want.items():
        if np.ptp(vals) == 0 and fn in ("CORR", "REGR_SLOPE", "REGR_INTERCEPT", "REGR_R2"):
            w = None
        # x is the first argument of the reference; the REGR_* functions regress y on x
        assert close(R.aggregate(fn, pa.float64(), x, ys=y), w, rel=1e-7), fn
    assert R.aggregate("REGR_COUNT", pa.float64(), [1.0, None, 2.0], ys=[None, 1.0, 2.0]) == 1


@pytest.mark.parametrize("vals", GROUPS, ids=lambda v: str(len(v)))
def test_percentiles_match_numpy(vals):
    x = vals.tolist()
    for q in (0.0, 0.1, 0.5, 0.99, 1.0):
        assert close(R.aggregate("PERCENTILE_CONT", pa.float64(), x, q=q), float(np.quantile(vals, q)))
        assert R.aggregate("PERCENTILE_DISC", pa.float64(), x, q=q) == np.quantile(vals, q, method="inverted_cdf")


def test_integer_sum_wraps_and_min_max_are_signed():
    assert R.aggregate("SUM", pa.int64(), [2**63 - 1, 1]) == -(2**63)
    assert R.aggregate("SUM", pa.int64(), [2**63 - 1, 2**63 - 1, 5]) == 3
    assert R.aggregate("SUM", pa.int8(), [127, 127]) == 254  # the sum is int64
    assert R.aggregate("MIN", pa.int64(), [-(2**63), 2**63 - 1]) == -(2**63)


def test_float_min_max_follow_total_order_and_keep_bits():
    nan_neg = og.float_of(0xFFF8000000000001 - (1 << 64))
    nan_pos = og.float_of(0x7FF0000000000001)
    vals = [1.0, nan_pos, -math.inf, nan_neg, -0.0, 0.0]
    assert R.bits(R.aggregate("MIN", pa.float64(), vals)) == R.bits(nan_neg)
    assert R.bits(R.aggregate("MAX", pa.float64(), vals)) == R.bits(nan_pos)
    assert R.bits(R.aggregate("MIN", pa.float64(), [0.0, -0.0])) == R.bits(-0.0)
    assert R.bits(R.aggregate("MAX", pa.float64(), [-0.0, 0.0])) == R.bits(0.0)
    assert math.isnan(R.aggregate("SUM", pa.float64(), [1.0, nan_pos]))
    assert R.aggregate("SUM", pa.float64(), [1.7976931348623157e308] * 2) == math.inf
    assert R.aggregate("PERCENTILE_DISC", pa.float64(), [nan_pos, 2.0, 1.0], q=1.0) == 2.0  # NaN is NULL


def test_canonical_reads_storage_of_edge_types():
    assert R.canonical(pa.array([2**64 - 1, 2**63, None], pa.uint64())) == [-1, -(2**63), None]
    assert R.canonical(pa.array([65535], pa.uint16())) == [65535]
    f16 = R.canonical(pa.array(np.array([65504, 2.0 ** -24, -0.0, np.nan], np.float16)))
    assert f16[:2] == [65504.0, 2.0 ** -24] and R.bits(f16[2]) == R.bits(-0.0) and math.isnan(f16[3])
    assert R.canonical(pa.array([datetime.date(1969, 12, 31)], pa.date32())) == [-1]
    assert R.canonical(pa.array([-1000], pa.date64())) == [-1000]
    assert R.canonical(pa.array([-5, 7], pa.timestamp("ns", "Europe/Berlin"))) == [-5, 7]
    assert R.canonical(pa.array([True, None, False])) == [1, None, 0]
    assert R.canonical(pa.array(["", "é", None]).dictionary_encode()) == ["", "é", None]


def test_uint64_follows_its_int64_bit_pattern_but_percentiles_order_unsigned():
    """DESIGN §7e: MIN sees 2^63 as INT64_MIN; the quantile kernel orders uint64 as unsigned."""
    vals = R.canonical(pa.array([1, 2**63, 3], pa.uint64()))
    assert R.aggregate("MIN", pa.uint64(), vals) == -(2**63)
    assert R.aggregate("PERCENTILE_DISC", pa.uint64(), vals, q=0.0) == 1
    assert R.aggregate("PERCENTILE_CONT", pa.uint64(), vals, q=1.0) == float(2**63)


def test_rejections_and_overflow():
    assert R.aggregate("SUM", pa.string(), ["a"]) is R.REJECTED
    assert R.aggregate("VAR_SAMP", pa.date32(), [1, 2]) is R.REJECTED
    assert R.aggregate("CORR", pa.bool_(), [1, 0], ys=[1.0, 2.0]) is R.REJECTED
    assert R.aggregate("PERCENTILE_CONT", pa.timestamp("s"), [1], q=0.5) is R.REJECTED
    assert R.aggregate("MIN", pa.string(), ["b", "", "é"]) == ""
    big = [1.7976931348623157e308, -1.7976931348623157e308]
    assert R.aggregate("VAR_POP", pa.float64(), big) is R.OVERFLOW
    assert R.aggregate("VAR_SAMP", pa.float64(), big[:1]) is None
    assert R.aggregate("REGR_COUNT", pa.float64(), big, ys=big) == 2
    # REGR_AVGX follows AVG: the float64 sum of [DBL_MAX, DBL_MAX, -1, 2] overflows, though the exact mean does not
    over = [1.7976931348623157e308, 1.7976931348623157e308, -1.0, 2.0]
    assert R.aggregate("REGR_AVGX", pa.float64(), over, ys=[0.0] * 4) == math.inf
    assert R.aggregate("REGR_AVGY", pa.float64(), [0.0] * 4, ys=over) == R.aggregate("AVG", pa.float64(), over)
    assert all(R.rejects(fn, pa.string()) == (AGGREGATES[fn].family not in ("basic", "pick")
                                               or fn in ("SUM", "AVG") or fn == "PERCENTILE_CONT")
               for fn in AGGREGATES if fn not in ("COUNT", "PERCENTILE_DISC"))
