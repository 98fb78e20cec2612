"""PERCENTILE_CONT / PERCENTILE_DISC / MEDIAN without a GPU: the exact reference (oracle/quantile.py) pinned
against pandas, numpy and hand-written values; the builders; the SQL forms; the multi-GPU decomposition."""
import math
import struct

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from fugue_b200.column import Kind, SelectColumns, col, functions as f, to_sql
from fugue_b200.execution_engine import decompose_aggs
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from oracle import quantile as Q


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _cont(values, q):
    t = pa.table({"v": pa.array(values, type=pa.float64())})
    return Q.quantiles_of(t, "v", np.arange(len(values)), [(q, Q.CONT)])[1][0]


# ---- the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("q", [0.0, 0.1, 0.25, 1 / 3, 0.5, 0.75, 0.9, 0.99, 1.0])
def test_cont_matches_pandas_groupby_quantile_bit_for_bit(q):
    rng = np.random.default_rng(7)
    n = 4000
    k = rng.integers(0, 150, n)
    v = rng.normal(0, 1e3, n)
    special = np.array([np.nan, np.inf, -np.inf, 1e308, -1e308, 5e-324, -5e-324, 2.2e-308, 0.0, 1.5])
    pick = rng.random(n) < 0.2
    v[pick] = special[rng.integers(0, len(special), pick.sum())]
    t = pa.table({"k": k, "v": v})
    want = pd.DataFrame({"k": k, "v": v}).groupby("k")["v"].quantile(q)
    got = Q.group_quantiles(t, ["k"], "v", [(q, Q.CONT)])
    for key, w in want.items():
        m, (r,) = got[(int(key),)]
        if m == 0:
            assert r is None and math.isnan(w)
        elif math.isnan(w):
            assert math.isnan(r)
        else:
            assert _bits(r) == _bits(w) or (r == 0 and w == 0), (key, r, w)


@pytest.mark.parametrize("q", [0.0, 0.3, 0.5, 0.77, 1.0])
def test_cont_matches_pandas_on_int64(q):
    rng = np.random.default_rng(3)
    k = rng.integers(0, 40, 2000)
    v = rng.integers(-(1 << 62), 1 << 62, 2000)
    t = pa.table({"k": k, "v": v})
    want = pd.DataFrame({"k": k, "v": v}).groupby("k")["v"].quantile(q)
    got = Q.group_quantiles(t, ["k"], "v", [(q, Q.CONT)])
    for key, w in want.items():
        assert _bits(got[(int(key),)][1][0]) == _bits(float(w))


@pytest.mark.parametrize("q", [0.0, 0.01, 0.2, 0.5, 0.51, 0.9, 1.0])
def test_disc_matches_numpy_inverted_cdf(q):
    rng = np.random.default_rng(5)
    for m in [1, 2, 3, 7, 10, 101]:
        v = rng.integers(-50, 50, m).astype(np.float64)
        t = pa.table({"v": v})
        _, (r,) = Q.quantiles_of(t, "v", np.arange(m), [(q, Q.DISC)])
        assert v[r] == np.quantile(v, q, method="inverted_cdf")


def test_hand_written_values():
    inf = math.inf
    assert _cont([1.0, 2.0, inf], 0.5) == 2.0  # the frac == 0 shortcut: no inf - inf
    assert math.isnan(_cont([-inf, inf], 0.5))
    assert _bits(_cont([-0.0, 0.0], 0.0)) == _bits(-0.0)  # ties keep row order
    assert _bits(_cont([0.0, -0.0], 0.0)) == _bits(0.0)
    assert _cont([-0.0, 0.0], 0.5) == 0.0
    assert _cont([4.0], 0.3) == 4.0  # m = 1
    assert _cont([], 0.5) is None and _cont([math.nan, None], 0.5) is None  # m = 0
    assert _cont([3.0, 1.0, 2.0], 0.0) == 1.0 and _cont([3.0, 1.0, 2.0], 1.0) == 3.0
    assert _cont([1.0, 2.0, 3.0, 4.0], 0.5) == 2.5
    t = pa.table({"v": pa.array([5.0, 5.0, 5.0])})
    assert Q.quantiles_of(t, "v", np.arange(3), [(0.5, Q.DISC)])[1] == [1]  # equal values: the tie-break by row
    assert Q.disc_position(0, 0.5) is None and Q.disc_position(4, 0.0) == 0 and Q.disc_position(4, 1.0) == 3


def test_uint64_converts_as_unsigned():
    t = pa.table({"v": pa.array([(1 << 63) + 2048, 1], type=pa.uint64())})
    assert Q.quantiles_of(t, "v", np.arange(2), [(1.0, Q.CONT)])[1] == [float((1 << 63) + 2048)]


def test_segments_and_groups_agree():
    t = pa.table({"k": [1, 1, 2, None, None, 2], "v": [3.0, 1.0, None, 2.0, 8.0, 4.0]})
    g = Q.group_quantiles(t, ["k"], "v", [(0.5, Q.CONT), (0.5, Q.DISC)])
    assert g[(1,)] == (2, [2.0, 1]) and g[(2,)] == (1, [4.0, 5]) and g[(None,)] == (2, [5.0, 3])
    m, res = Q.segment_quantiles(t, "v", np.array([0, 2, 2, 6]), [(0.5, Q.CONT)])
    assert list(m) == [2, 0, 3] and res[0] == [2.0, None, 4.0]


# ---- builders --------------------------------------------------------------------------------------
def test_builders():
    m = f.median(col("v"))
    assert m.kind == Kind.AGG and m.func == "PERCENTILE_CONT" and m.arg.name == "v" and m.kwargs == {"q": 0.5}
    assert m.fingerprint() == f.percentile_cont("v", 0.5).fingerprint() == f.percentile_cont(col("v"), 0.5).fingerprint()
    assert f.percentile_cont("v", 1).kwargs == {"q": 1.0} and isinstance(f.percentile_cont("v", 1).kwargs["q"], float)
    d = f.percentile_disc(col("v"), 0.9)
    assert d.func == "PERCENTILE_DISC" and d.kwargs == {"q": 0.9}
    assert f.percentile_cont("v", 0.25).infer_alias().output_name == "v"
    assert f.is_agg(d) and f.is_agg(f.median(col("a")) * 2)
    for bad in [-0.1, 1.5, math.nan, True, "0.5", None, math.inf]:
        with pytest.raises(ValueError):
            f.percentile_cont("v", bad)
        with pytest.raises(ValueError):
            f.percentile_disc("v", bad)
    with pytest.raises(ValueError):
        f.median(col("*"))
    with pytest.raises(ValueError):
        f.median(f.sum(col("v")))


def test_over():
    w = f.median(col("v")).over()
    assert w.kind == Kind.WINDOW and w.func == "PERCENTILE_CONT" and w.kwargs == {"q": 0.5}
    assert f.percentile_disc(col("v"), 0.3).over().kwargs == {"q": 0.3}
    for kw in [dict(running=True), dict(rows=(-1, 1)), dict(rows=(None, None)), dict(range=(None, None)),
               dict(range=(-1, 0))]:
        with pytest.raises(ValueError):
            f.median(col("v")).over(**kw)
    assert to_sql(w.alias("m")) == "PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY v) OVER () AS m"


def test_inferred_types():
    s = Schema("a:int,b:float,c:str,d:date,e:uint64")
    for c in "abcde":
        assert f.percentile_cont(col(c), 0.5).infer_type(s) == pa.float64()
        assert f.percentile_cont(col(c), 0.5).over().infer_type(s) == pa.float64()
        assert f.percentile_disc(col(c), 0.5).infer_type(s) == s[c].type
        assert f.percentile_disc(col(c), 0.5).over().infer_type(s) == s[c].type


# ---- SQL -------------------------------------------------------------------------------------------
def _parse(items, rest):
    return _parse_select(items, rest, f"SELECT {items} FROM {rest}")


def test_sql_forms():
    st = _parse("key, MEDIAN(v) AS m, PERCENTILE_CONT(0.9) WITHIN GROUP (ORDER BY v) p90, "
                "PERCENTILE_DISC(0.25) WITHIN GROUP (ORDER BY v ASC) AS d, QUANTILE_CONT(v, 0.1) AS qc, "
                "QUANTILE_DISC(v * 2, 1) qd, SUM(v) AS s",
                "t WHERE v > 0 GROUP BY key HAVING MEDIAN(v) > 1.5 ORDER BY m DESC")
    m, p90, d, qc, qd, s = st.columns[1:]
    assert m.fingerprint() == f.median(col("v")).alias("m").fingerprint()
    assert p90.fingerprint() == f.percentile_cont(col("v"), 0.9).alias("p90").fingerprint()
    assert d.fingerprint() == f.percentile_disc(col("v"), 0.25).alias("d").fingerprint()
    assert qc.fingerprint() == f.percentile_cont(col("v"), 0.1).alias("qc").fingerprint()
    assert qd.fingerprint() == f.percentile_disc(col("v") * 2, 1).alias("qd").fingerprint()
    assert [str(g) for g in st.group_by] == ["key"] and st.order_by == [("m", False)]
    assert str(st.having) == str(f.median(col("v")) > 1.5)
    st = _parse("PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY v)", "t")
    assert st.columns[0].output_name == "v" and st.group_by == []


def test_sql_rejections():
    with pytest.raises(NotImplementedError):
        _parse("PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY v DESC) AS m", "t")
    with pytest.raises(NotImplementedError):
        _parse("PERCENTILE_CONT(q) WITHIN GROUP (ORDER BY v) AS m", "t")
    with pytest.raises(NotImplementedError):
        _parse("PERCENTILE_CONT(0.5) AS m", "t")
    with pytest.raises(ValueError):
        _parse("QUANTILE_DISC(v, 2) AS m", "t")


@pytest.mark.parametrize("e", [f.median(col("v")).alias("m"), f.percentile_cont(col("a") + 1, 0.125).alias("x"),
                               f.percentile_disc(col("v"), 1).alias("d"), f.percentile_disc(col("v"), 0).alias("z"),
                               (f.median(col("v")) * 2 - f.sum(col("w"))).alias("y")])
def test_print_parse_round_trip(e):
    text = to_sql(e)
    st = _parse(text, "t")
    assert st.columns[0].fingerprint() == e.fingerprint(), text


def test_window_print_is_parseable_prefix():
    assert to_sql(f.percentile_disc(col("v"), 0.5).over()) == \
        "PERCENTILE_DISC(0.5) WITHIN GROUP (ORDER BY v) OVER ()"


# ---- engines -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("a", [f.median(col("v")).alias("m"), f.percentile_disc(col("v"), 0.5).alias("d")])
def test_no_partial_final_decomposition(a):
    with pytest.raises(NotImplementedError, match="has no partial / final decomposition"):
        decompose_aggs([a])


def test_select_list_roles():
    sc = SelectColumns(col("k"), f.median(col("v")).alias("m"))
    assert sc.has_agg and [str(g) for g in sc.group_keys] == ["k"]
