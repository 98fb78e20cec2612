"""SKEWNESS / SKEWNESS_POP / KURTOSIS / KURTOSIS_POP without a GPU: builders, aliases, type inference, the SQL
names and their round trip, the DISTINCT / frame / multi-GPU / string and boolean rejections, the accumulator plan of
the hash group-by, the finisher's NULL / constant / NaN rules, the host side of K6's correction and a float64 model of
K9's pairwise update against the exact reference (oracle/shape_moments.py), and that reference against pandas and
scipy."""
import math
import types
from typing import List

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import scipy.stats
import torch

from fugue_b200 import aggregates as A
from fugue_b200 import kernels as K
from fugue_b200.column import SHAPES, VARIANCES, Kind, SelectColumns, agg, col, functions as f, to_sql
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.dist import DistributedB200Engine
from fugue_b200.execution_engine import B200ExecutionEngine, decompose_aggs
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table
from oracle import shape_moments as OS

BUILDERS = [(f.skewness, "SKEWNESS"), (f.skew, "SKEWNESS"), (f.skewness_pop, "SKEWNESS_POP"),
            (f.kurtosis, "KURTOSIS"), (f.kurt, "KURTOSIS"), (f.kurtosis_pop, "KURTOSIS_POP")]
SQL_NAMES = {"SKEWNESS": "SKEWNESS", "SKEW": "SKEWNESS", "SKEWNESS_POP": "SKEWNESS_POP", "KURTOSIS": "KURTOSIS",
             "KURT": "KURTOSIS", "KURTOSIS_POP": "KURTOSIS_POP"}
SHAPE_OPS = [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64, K.AGG_DEV3_F64, K.AGG_DEV4_F64, K.AGG_MIN_F64,
             K.AGG_MAX_F64]


# ---- IR ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("build,head", BUILDERS)
def test_builders_give_canonical_heads(build, head):
    e = build(col("v"))
    assert e.kind == Kind.AGG and e.func == head and e.arg.name == "v" and not e.is_distinct
    assert e.fingerprint() == build("v").fingerprint() == agg(head.lower(), "v").fingerprint()
    assert e.infer_alias().output_name == "v"
    assert f.is_agg(e) and f.is_agg(e * 2 + 1)


def test_family_is_its_own():
    assert SHAPES == {"SKEWNESS", "SKEWNESS_POP", "KURTOSIS", "KURTOSIS_POP"}
    assert VARIANCES == {"VAR_SAMP", "VAR_POP", "STDDEV_SAMP", "STDDEV_POP"}


def test_aliases_of_agg():
    assert agg("skew", "v").func == "SKEWNESS" and agg("Kurt", "v").func == "KURTOSIS"
    assert agg("kurtosis_pop", "v").func == "KURTOSIS_POP"


def test_inferred_type_is_float64():
    s = Schema("a:int,b:double,c:uint8,d:float16,e:long")
    for c in s.names:
        for build, _ in BUILDERS:
            assert build(col(c)).infer_type(s) == pa.float64()
            assert build(col(c)).over().infer_type(s) == pa.float64()
            assert build(col(c)).over(running=True).infer_type(s) == pa.float64()


def test_over_forms():
    w = f.skew(col("v")).over()
    assert w.kind == Kind.WINDOW and w.func == "SKEWNESS" and w.kwargs == {"running": False}
    assert f.kurtosis_pop(col("v")).over(running=True).kwargs == {"running": True}
    assert f.kurt(col("v")).over(rows=(None, 0)).kwargs == {"running": True}
    assert f.kurt(col("v")).over(range=(None, None)).kwargs == {"running": False}
    assert to_sql(w.alias("s")) == "SKEWNESS(v) OVER () AS s"


@pytest.mark.parametrize("kw", [{"rows": (-3, 0)}, {"rows": (0, 2)}, {"range": (-1, 1)}, {"range": (None, 0)}])
def test_frames_are_not_supported(kw):
    for build, _ in BUILDERS:
        with pytest.raises(NotImplementedError, match="ROWS and RANGE frames are not supported"):
            build(col("v")).over(**kw)


def test_distinct_is_rejected():
    with pytest.raises(ValueError):
        agg("KURTOSIS", "v", arg_distinct=True).over()
    with pytest.raises(NotImplementedError, match="DISTINCT"):
        _parse("SKEW(DISTINCT v) AS s", "t")


# ---- SQL ---------------------------------------------------------------------------------------------
def _parse(items, rest):
    return _parse_select(items, rest, f"SELECT {items} FROM {rest}")


@pytest.mark.parametrize("name", sorted(SQL_NAMES))
def test_sql_names(name):
    for spelled in (name, name.lower(), name.capitalize()):
        st = _parse(f"key, {spelled}(v) AS s, {spelled}(v * 2 + w) x", "t GROUP BY key HAVING " + spelled + "(v) > 1")
        s, x = st.columns[1:]
        assert s.func == SQL_NAMES[name] and s.output_name == "s" and s.arg.name == "v"
        assert x.fingerprint() == agg(SQL_NAMES[name], col("v") * 2 + col("w")).alias("x").fingerprint()
        assert st.having.left.func == SQL_NAMES[name]


@pytest.mark.parametrize("e", [f.skew(col("v")).alias("s"), f.kurt(col("a") + 1).alias("x"),
                               f.skewness_pop(col("v")).alias("p"), f.kurtosis_pop(col("v") * col("w")).alias("q"),
                               (f.kurtosis(col("v")) - f.skewness(col("v"))).alias("d"),
                               f.skewness(col("v")).cast("float").alias("c")])
def test_print_parse_fixed_point(e):
    text = to_sql(e)
    st = _parse(text, "t")
    assert st.columns[0].fingerprint() == e.fingerprint(), text
    assert to_sql(st.columns[0]) == text


# ---- engine plans ------------------------------------------------------------------------------------
def test_no_partial_final_decomposition():
    for build, _ in BUILDERS:
        with pytest.raises(NotImplementedError, match="has no partial / final decomposition"):
            decompose_aggs([build(col("v")).alias("s")])
        with pytest.raises(NotImplementedError):
            decompose_aggs([f.count(col("v")).alias("c"), build(col("v")).alias("s")])


def test_multi_gpu_raises_before_device_work():
    t = B200Table(Schema("k:long,v:double"), [torch.tensor([1, 2]), torch.tensor([1.0, 2.0])])
    fake = types.SimpleNamespace(_world=2, to_df=lambda df: df, _plain_aggs=B200ExecutionEngine._plain_aggs)
    for build, _ in BUILDERS:
        for spec in (PartitionSpec(by=["k"]), None):
            with pytest.raises(NotImplementedError):
                DistributedB200Engine.aggregate(fake, B200DataFrame(t), spec, [build(col("v")).alias("s")])


def test_plain_aggs_take_the_family():
    assert B200ExecutionEngine._plain_aggs([b(col("v")).alias("s") for b, _ in BUILDERS])
    assert not B200ExecutionEngine._plain_aggs([f.skew(col("v") + 1).alias("s")])


class _Spy:
    """Replaces ``kernels.groupby_u64``: records the accumulators and returns one group of zeros."""

    def __init__(self, monkeypatch):
        self.calls = []

        def groupby(keys, kv, vals, vv, ops, **kw):
            self.calls.append((list(vals), list(vv), list(ops)))
            z = torch.zeros(1, dtype=torch.int64)
            return z, None if kv is None else torch.ones(1, dtype=torch.uint8), [z.clone() for _ in ops], 1

        monkeypatch.setattr(K, "groupby_u64", groupby)


def _named(t, keys, aggs, monkeypatch):
    spy = _Spy(monkeypatch)
    fake = types.SimpleNamespace(to_df=lambda df: df, _aggregate_sorted=lambda *a: "sorted",
                                 _pair_accumulators=B200ExecutionEngine._pair_accumulators,
                                 _pair_moments=B200ExecutionEngine._pair_moments)
    res = B200ExecutionEngine._aggregate_named(fake, B200DataFrame(t), PartitionSpec(by=keys) if keys else None, aggs)
    return res if res == "sorted" else spy.calls[-1]


def _t():
    return B200Table(Schema("k:long,v:double,w:int,x:float"),
                     [torch.tensor([1, 2]), torch.tensor([1.0, 2.0]), torch.tensor([3, 4], dtype=torch.int32),
                      torch.tensor([5.0, 6.0], dtype=torch.float32)],
                     [None, torch.tensor([1, 0], dtype=torch.uint8), None, None])


def test_one_set_per_column_shared_with_the_variances(monkeypatch):
    t = _t()
    vals, vv, ops = _named(t, ["k"], [b(col("v")).alias(f"s{i}") for i, (b, _) in enumerate(BUILDERS)], monkeypatch)
    assert ops == SHAPE_OPS
    assert vals[1] is None and all(x is vals[0] for i, x in enumerate(vals) if i != 1)
    assert vals[0].dtype == torch.float64 and all(m is t.valid[1] for m in vv)
    # a variance first, then a shape statistic of the same column: the variance's four and the four more
    _, _, ops = _named(t, ["k"], [f.stddev(col("v")).alias("a"), f.kurt(col("v")).alias("b"),
                                  f.var_pop(col("v")).alias("c"), f.skew(col("v")).alias("d")], monkeypatch)
    assert ops == SHAPE_OPS
    # a variance of one column and a shape statistic of another: one set each
    vals, vv, ops = _named(t, ["k"], [f.stddev(col("w")).alias("a"), f.skew(col("v")).alias("b")], monkeypatch)
    assert ops == SHAPE_OPS[:4] + SHAPE_OPS and vals[0].tolist() == [3.0, 4.0] and vv[:4] == [None] * 4
    # a global aggregate takes the same accumulators (its COUNT also gives the NULL of an empty input)
    _, _, ops = _named(t, [], [f.kurtosis_pop(col("x")).alias("a")], monkeypatch)
    assert ops == SHAPE_OPS


def test_a_pair_and_a_shape_statistic_share_the_column_set(monkeypatch):
    t = _t()
    vals, _, ops = _named(t, ["k"], [f.skew(col("w")).alias("a"), f.corr(col("w"), col("x")).alias("b")], monkeypatch)
    # w's eight, then the pair's: SUM y, CODEV, DEV y, DEV2 y, MIN / MAX of x and y (x reuses w's set)
    assert ops[:8] == SHAPE_OPS and ops.count(K.AGG_SUM_F64) == 2 and ops.count(K.AGG_DEV3_F64) == 1
    assert len(ops) == 16


def test_capacity_takes_the_sorted_route(monkeypatch):
    t = _t()
    # two columns of eight fill one kernel call
    _, _, ops = _named(t, ["k"], [f.kurt(col("v")).alias("a"), f.skew(col("w")).alias("b")], monkeypatch)
    assert len(ops) == K.MAX_AGGS
    # a third column does not fit: the sorted route, which has no such limit
    assert _named(t, ["k"], [f.kurt(col("v")).alias("a"), f.skew(col("w")).alias("b"), f.skew(col("x")).alias("c")],
                  monkeypatch) == "sorted"


@pytest.mark.parametrize("schema,col_", [("k:long,s:bool", torch.tensor([1, 0], dtype=torch.uint8)),
                                         ("k:long,s:str", torch.tensor([0, 1], dtype=torch.int32))])
def test_strings_and_booleans_raise(schema, col_, monkeypatch):
    t = B200Table(Schema(schema), [torch.tensor([1, 2]), col_], None,
                  {"s": pa.array(["x", "y"])} if schema.endswith("str") else {})
    for build, _ in BUILDERS:
        with pytest.raises(NotImplementedError, match="needs integer or float columns"):
            _named(t, ["k"], [build(col("s")).alias("a")], monkeypatch)


@pytest.mark.parametrize("fn", sorted(SHAPES))
@pytest.mark.parametrize("tp,is_dict", [(pa.string(), True), (pa.bool_(), False), (pa.date32(), False)])
def test_check_argument_rejects(fn, tp, is_dict):
    with pytest.raises(NotImplementedError):
        A.check_argument(fn, "a", tp, is_dict)


# ---- the finisher ------------------------------------------------------------------------------------
def _f(*xs):
    return torch.tensor(xs, dtype=torch.float64)


def test_null_rules_by_count():
    m = torch.tensor([0, 1, 2, 3, 4, 5])
    m2, m3, m4 = _f(0, 0, 2, 2, 5, 10), _f(0, 0, 0, 1, 3, 4), _f(0, 0, 2, 3, 7, 30)
    want = {"SKEWNESS": 3, "SKEWNESS_POP": 1, "KURTOSIS": 4, "KURTOSIS_POP": 1}
    for fn, need in want.items():
        v, ok = A.shape_of(fn, m, m2, m3, m4)
        assert ok.tolist() == [int(c >= need) for c in m.tolist()]
        assert v.dtype == torch.float64 and all(x == 0 for x, o in zip(v.tolist(), ok.tolist()) if not o)


def test_constant_group_is_zero_and_nan_propagates():
    m = torch.tensor([6, 6, 6])
    m2, m3, m4 = _f(0, math.nan, 4), _f(0, math.nan, math.nan), _f(0, math.nan, 5)
    for fn in SHAPES:
        v, ok = A.shape_of(fn, m, m2, m3, m4)
        assert ok.tolist() == [1, 1, 1] and v[0].item() == 0.0 and math.isnan(v[1].item())
    # a NaN M3 or M4 beside a finite M2 reaches only the statistic that reads it
    assert math.isnan(A.shape_of("SKEWNESS", m, m2, m3, m4)[0][2].item())
    assert not math.isnan(A.shape_of("KURTOSIS", m, m2, m3, m4)[0][2].item())


@pytest.mark.parametrize("fn", sorted(SHAPES))
def test_finisher_matches_the_exact_finish(fn):
    rng = np.random.default_rng(1)
    for m in (4, 5, 9, 100, 1000):
        v = rng.gamma(1.5, 2.0, m).tolist()
        mm, *q = OS.central_sums(v)
        got, ok = A.shape_of(fn, torch.tensor([mm]), *(_f(float(x)) for x in q))
        want = OS.finish(fn, (mm, *q))
        scale = abs(want) + 3 * (m - 1) ** 2 / ((m - 2) * (m - 3)) if fn == "KURTOSIS" else abs(want) + 3
        assert ok.item() == 1 and abs(got.item() - want) <= 8 * OS.U * scale, (m, got.item(), want)


def _gaggs(v: List[float], c: float):
    """The eight K6 accumulators of one group of values ``v`` as K6 leaves them when its summed mean is ``c``."""
    x = np.asarray(v, dtype=np.float64)
    d = x - c  # exact: c is within a factor 2 of every x here
    sums = [float(np.sum(d ** k)) for k in (1, 2, 3, 4)]
    bits = [torch.tensor([s], dtype=torch.float64).view(torch.int64) for s in
            [float(np.sum(x))] + sums + [float(x.min()), float(x.max())]]
    return [bits[0], torch.tensor([len(v)])] + bits[1:]


def test_shape_moments_correct_a_shifted_mean():
    rng = np.random.default_rng(2)
    for shift, sigma in ((0.0, 1.0), (1e6, 3.0), (1e9, 1e-3)):
        v = (shift + sigma * rng.standard_normal(500) ** 3).tolist()
        mean = float(np.mean(v))
        # a summed mean 64 u m |x| off, the worst the atomics give
        c = mean + 64 * len(v) * OS.U * max(abs(x) for x in v) * 0.5
        m, *got = A.shape_moments(_gaggs(v, c), tuple(range(8)))
        _, *ex = OS.central_sums(v)
        bounds = OS.sums_bound(v, "hash")
        assert m.item() == len(v)
        for g, e, b in zip(got, ex, bounds):
            assert abs(g.item() - float(e)) <= b * 64, (shift, g.item(), float(e), b)


def test_shape_moments_constant_and_non_finite():
    g = _gaggs([0.1] * 7, 0.1 * 7 / 7 + 1e-17)
    assert [q.item() for q in A.shape_moments(g, tuple(range(8)))[1:]] == [0.0, 0.0, 0.0]
    for bad in (math.nan, math.inf, -math.inf):
        g = _gaggs([1.0, 2.0, 4.0], 7 / 3)
        g[6 if bad != math.inf else 7] = torch.tensor([bad], dtype=torch.float64).view(torch.int64)
        assert all(math.isnan(q.item()) for q in A.shape_moments(g, tuple(range(8)))[1:])


# ---- a float64 model of K9's update ------------------------------------------------------------------
def _combine(a, b):
    """Pebay's pairwise update of (n, mean, M2, M3, M4), written as fb_window.cu writes it (nb / n by one
    division here, within the same 2 u)."""
    if b[0] == 0:
        return a
    if a[0] == 0:
        return b
    na, ma, a2, a3, a4 = a
    nb, mb, b2, b3, b4 = b
    n = na + nb
    wa, wb = na / n, nb / n
    d = mb - ma
    d2 = d * d
    t2 = d2 * na * wb
    return (n, ma + d * wb, a2 + b2 + t2, a3 + b3 + t2 * d * (wa - wb) + 3.0 * d * (wa * b2 - wb * a2),
            a4 + b4 + t2 * d2 * (wa * wa - wa * wb + wb * wb) + 6.0 * d2 * (wa * wa * b2 + wb * wb * a2)
            + 4.0 * d * (wa * b3 - wb * a3))


def _tree(states):
    while len(states) > 1:
        states = [_combine(states[i], states[i + 1]) if i + 1 < len(states) else states[i]
                  for i in range(0, len(states), 2)]
    return states[0]


@pytest.mark.parametrize("order", ["sequential", "tree"])
def test_pairwise_update_model_meets_the_scan_bound(order):
    rng = np.random.default_rng(3)
    for m, mean, sigma in ((5, 0.0, 1.0), (300, 50.0, 5.0), (2000, -1e4, 2.0)):
        v = (mean + sigma * rng.gamma(2.0, 1.0, m)).tolist()
        states = [(1, x, 0.0, 0.0, 0.0) for x in v]
        st = _tree(states) if order == "tree" else states[0]
        if order == "sequential":
            for s in states[1:]:
                st = _combine(st, s)
        _, *ex = OS.central_sums(v)
        for g, e, b in zip(st[2:], ex, OS.sums_bound(v, "scan")):
            assert abs(g - float(e)) <= b, (m, g, float(e), b)
    # equal values: every delta is exactly 0
    st = _tree([(1, 0.1, 0.0, 0.0, 0.0)] * 37)
    assert st[2:] == (0.0, 0.0, 0.0)


# ---- the reference -----------------------------------------------------------------------------------
def test_oracle_against_pandas_and_scipy():
    rng = np.random.default_rng(5)
    for m in (4, 5, 17, 200, 3000):
        for v in (rng.standard_normal(m), rng.gamma(2.0, 3.0, m) - 4.0, rng.standard_t(5, m) * 100 + 7):
            vals = v.tolist()
            s = pd.Series(v)
            checks = {"SKEWNESS": (s.skew(), scipy.stats.skew(v, bias=False)),
                      "SKEWNESS_POP": (scipy.stats.skew(v, bias=True),),
                      "KURTOSIS": (s.kurt(), scipy.stats.kurtosis(v, bias=False)),
                      "KURTOSIS_POP": (scipy.stats.kurtosis(v, bias=True),)}
            for fn, others in checks.items():
                r = OS.result(fn, vals)
                for o in others:
                    # pandas and scipy sum in float64: within their rounding of the exact value
                    assert math.isclose(r, o, rel_tol=1e-10, abs_tol=1e-12), (fn, m, r, o)


def test_oracle_grouped_against_pandas():
    rng = np.random.default_rng(6)
    n = 4000
    k = rng.integers(0, 60, n)
    v = rng.normal(3.0, 2.0, n)
    v[rng.random(n) < 0.1] = np.nan  # pandas' NaN is NULL here
    df = pd.DataFrame({"k": k, "v": v})
    vals = [None if math.isnan(x) else x for x in v.tolist()]
    for fn, want in (("SKEWNESS", df.groupby("k")["v"].skew()),
                     ("KURTOSIS", df.groupby("k")["v"].apply(lambda s: s.kurt()))):
        got = OS.group_results(fn, k.tolist(), vals)
        for key, x in want.items():
            r = got[int(key)]
            assert (r is None) if math.isnan(x) else math.isclose(r, x, rel_tol=1e-10), (fn, key, r, x)


def test_oracle_edges():
    for fn in SHAPES:
        assert OS.result(fn, []) is None and OS.result(fn, [None, None]) is None
        assert OS.result(fn, [5.0] * 4) == 0.0  # pandas: [5, 5, 5, 5].skew() == kurt() == 0
        for bad in (math.nan, math.inf, -math.inf):
            assert math.isnan(OS.result(fn, [1.0, bad, 2.0, 7.0]))
    assert OS.result("SKEWNESS", [1.0, 2.0]) is None and OS.result("SKEWNESS", [1.0, 2.0, 4.0]) is not None
    assert OS.result("KURTOSIS", [1.0, 2.0, 4.0]) is None
    assert OS.result("SKEWNESS_POP", [3.0]) == 0.0 and OS.result("KURTOSIS_POP", [3.0]) == 0.0
    assert OS.result("SKEWNESS", [0.0, 0.0, 3.0]) == pytest.approx(math.sqrt(3))  # G1 of (0, 0, 3): sqrt(3)
    assert OS.result("KURTOSIS_POP", [-1.0, 1.0]) == -2.0
    # the running and whole-partition forms
    assert OS.running_results("SKEWNESS_POP", [None, 1.0, 1.0]) == [None, 0.0, 0.0]
    assert OS.partition_results("KURTOSIS_POP", [-1.0, None, 1.0]) == [-2.0] * 3
    # pandas zeroes central sums it takes for rounding noise (below (eps max|x|)^k m); the exact reference does not
    near = [1e9, 1e9, 1e9, math.nextafter(1e9, math.inf)]
    assert OS.result("SKEWNESS", near) == 2.0 and pd.Series(near).skew() == 0.0


def test_naive_power_sums_fail_at_a_high_mean():
    rng = np.random.default_rng(7)
    v = (1e9 + 1e-3 * rng.standard_normal(1000)).tolist()
    for fn in SHAPES:
        assert abs(OS.naive_power_sums(fn, v) - OS.result(fn, v)) > OS.result_bound(fn, v, "hash")
