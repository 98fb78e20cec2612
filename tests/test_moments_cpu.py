"""VAR_SAMP / VAR_POP / STDDEV_SAMP / STDDEV_POP without a GPU: builders, type inference, the SQL forms and
their round trip, the frame and DISTINCT rejections, the multi-GPU and COUNT(DISTINCT) rejections, the
accumulator plan of the hash group-by, and the exact reference (oracle/moments.py) pinned to ``statistics``
and pandas."""
import math
import statistics
import types

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

from fugue_b200 import kernels as K
from fugue_b200.column import VARIANCES, Kind, SelectColumns, agg, col, functions as f, to_sql
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.dist import DistributedB200Engine
from fugue_b200.execution_engine import B200ExecutionEngine, decompose_aggs
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table
from oracle import moments as OM

BUILDERS = [(f.var_samp, "VAR_SAMP"), (f.variance, "VAR_SAMP"), (f.var_pop, "VAR_POP"),
            (f.stddev_samp, "STDDEV_SAMP"), (f.stddev, "STDDEV_SAMP"), (f.stddev_pop, "STDDEV_POP")]
SQL_NAMES = {"VAR_SAMP": "VAR_SAMP", "VARIANCE": "VAR_SAMP", "VAR_POP": "VAR_POP", "STDDEV_SAMP": "STDDEV_SAMP",
             "STDDEV": "STDDEV_SAMP", "STDDEV_POP": "STDDEV_POP"}


# ---- IR ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("build,head", BUILDERS)
def test_builders_give_canonical_heads(build, head):
    e = build(col("v"))
    assert e.kind == Kind.AGG and e.func == head and e.arg.name == "v" and not e.is_distinct
    assert e.fingerprint() == build("v").fingerprint() == agg(head.lower(), "v").fingerprint()
    assert e.infer_alias().output_name == "v"
    assert f.is_agg(e) and f.is_agg(e * 2 + 1)
    assert VARIANCES == {"VAR_SAMP", "VAR_POP", "STDDEV_SAMP", "STDDEV_POP"}


def test_aliases_of_agg():
    assert agg("stddev", "v").func == "STDDEV_SAMP" and agg("Variance", "v").func == "VAR_SAMP"


def test_inferred_type_is_float64():
    s = Schema("a:int,b:double,c:uint8,d:float16,e:long")
    for c in s.names:
        for build, _ in BUILDERS:
            assert build(col(c)).infer_type(s) == pa.float64()
            assert build(col(c)).over().infer_type(s) == pa.float64()
            assert build(col(c)).over(running=True).infer_type(s) == pa.float64()


def test_over_forms():
    w = f.stddev(col("v")).over()
    assert w.kind == Kind.WINDOW and w.func == "STDDEV_SAMP" and w.kwargs == {"running": False}
    assert f.var_pop(col("v")).over(running=True).kwargs == {"running": True}
    # the spellings of the whole partition and of the running frame give those nodes
    assert f.var_pop(col("v")).over(rows=(None, 0)).kwargs == {"running": True}
    assert f.var_pop(col("v")).over(rows=(None, None)).kwargs == {"running": False}
    assert f.var_pop(col("v")).over(range=(None, None)).kwargs == {"running": False}
    assert to_sql(w.alias("s")) == "STDDEV_SAMP(v) OVER () AS s"


@pytest.mark.parametrize("kw", [{"rows": (-3, 0)}, {"rows": (0, 2)}, {"rows": (None, 1)}, {"range": (-1, 1)},
                                {"range": (None, 0)}])
def test_frames_are_not_supported(kw):
    for build, _ in BUILDERS:
        with pytest.raises(NotImplementedError, match="ROWS and RANGE frames are not supported"):
            build(col("v")).over(**kw)


def test_distinct_is_rejected():
    with pytest.raises(ValueError):
        agg("STDDEV_SAMP", "v", arg_distinct=True).over()
    with pytest.raises(NotImplementedError, match="DISTINCT"):
        _parse("STDDEV(DISTINCT v) AS s", "t")


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


@pytest.mark.parametrize("e", [f.stddev(col("v")).alias("s"), f.variance(col("a") + 1).alias("x"),
                               f.var_pop(col("v")).alias("p"), f.stddev_pop(col("v") * col("w")).alias("q"),
                               (f.stddev(col("v")) / f.avg(col("v"))).alias("cv"),
                               f.var_samp(col("v")).cast("float").alias("c")])
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
        # COUNT(DISTINCT x) in the same SELECT goes through the same decomposition
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
    assert not B200ExecutionEngine._plain_aggs([f.stddev(col("v") + 1).alias("s")])


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
    fake = types.SimpleNamespace(to_df=lambda df: df)
    B200ExecutionEngine._aggregate_named(fake, B200DataFrame(t), PartitionSpec(by=keys) if keys else None, aggs)
    return spy.calls[-1]


def test_four_accumulators_per_column_shared(monkeypatch):
    t = B200Table(Schema("k:long,v:double,w:int"), [torch.tensor([1, 2]), torch.tensor([1.0, 2.0]),
                                                    torch.tensor([3, 4], dtype=torch.int32)],
                  [None, torch.tensor([1, 0], dtype=torch.uint8), None])
    vals, vv, ops = _named(t, ["k"], [b(col("v")).alias(f"s{i}") for i, (b, _) in enumerate(BUILDERS)], monkeypatch)
    assert ops == [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64]
    assert vals[0] is vals[2] is vals[3] and vals[1] is None and vals[0].dtype == torch.float64
    assert all(m is t.valid[1] for m in vv)
    vals, vv, ops = _named(t, ["k"], [f.stddev(col("v")).alias("a"), f.var_pop(col("w")).alias("b"),
                                      f.stddev_pop(col("v")).alias("c")], monkeypatch)
    assert ops == [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64] * 2
    assert vals[4].dtype == torch.float64 and vals[4].tolist() == [3.0, 4.0] and vv[4:] == [None] * 4
    # a global aggregate: the same four (the COUNT also gives the NULL of an empty input)
    _, _, ops = _named(t, [], [f.stddev(col("w")).alias("a")], monkeypatch)
    assert ops == [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64]


@pytest.mark.parametrize("schema,col_", [("k:long,s:bool", torch.tensor([1, 0], dtype=torch.uint8)),
                                         ("k:long,s:str", torch.tensor([0, 1], dtype=torch.int32))])
def test_strings_and_booleans_raise(schema, col_, monkeypatch):
    t = B200Table(Schema(schema), [torch.tensor([1, 2]), col_], None,
                  {"s": pa.array(["x", "y"])} if schema.endswith("str") else {})
    for build, _ in BUILDERS:
        with pytest.raises(NotImplementedError):
            _named(t, ["k"], [build(col("s")).alias("a")], monkeypatch)


def test_select_list_roles():
    sc = SelectColumns(col("k"), f.stddev(col("v")).alias("s"))
    assert sc.has_agg and [str(g) for g in sc.group_keys] == ["k"]


# ---- the reference -----------------------------------------------------------------------------------
def _fn(fn, vals):
    return OM.result(fn, *OM.moments(vals))


def test_oracle_against_statistics():
    rng = np.random.default_rng(11)
    for m in [2, 3, 5, 17, 200]:
        for scale, shift in [(1.0, 0.0), (1e-3, 1e9), (1e10, -3.0), (1.0, 1e15)]:
            v = (rng.standard_normal(m) * scale + shift).tolist()
            # statistics divides the exact M2 and rounds once: so does result_exact
            assert OM.result_exact("VAR_SAMP", v) == statistics.variance(v)
            assert OM.result_exact("VAR_POP", v) == statistics.pvariance(v)
            assert math.isclose(OM.result_exact("STDDEV_SAMP", v), statistics.stdev(v), rel_tol=2 ** -52)
            assert math.isclose(OM.result_exact("STDDEV_POP", v), statistics.pstdev(v), rel_tol=2 ** -52)
            # the rounded M2 divided once more: within one more rounding (u = 2^-53)
            for fn in OM.FUNCS:
                assert math.isclose(_fn(fn, v), OM.result_exact(fn, v), rel_tol=2 * 2 ** -53)


def test_oracle_against_pandas():
    rng = np.random.default_rng(5)
    n = 3000
    k = rng.integers(0, 120, n)
    v = rng.normal(3.0, 2.0, n)
    v[rng.random(n) < 0.1] = np.nan  # pandas' NaN is NULL here
    df = pd.DataFrame({"k": k, "v": v})
    want = {"VAR_SAMP": df.groupby("k")["v"].var(), "VAR_POP": df.groupby("k")["v"].var(ddof=0),
            "STDDEV_SAMP": df.groupby("k")["v"].std(), "STDDEV_POP": df.groupby("k")["v"].std(ddof=0)}
    got = OM.group_moments(k.tolist(), [None if math.isnan(x) else x for x in v])
    for fn, w in want.items():
        for key, x in w.items():
            r = OM.result(fn, *got[int(key)])
            if math.isnan(x):
                assert r is None
            else:
                # pandas sums in a different order: within a few ulp of the correctly rounded result
                assert math.isclose(r, x, rel_tol=1e-13), (fn, key, r, x)


def test_oracle_edges():
    assert OM.moments([]) == (0, None) and OM.moments([None]) == (0, None)
    assert OM.moments([2.5]) == (1, 0.0)
    assert _fn("VAR_SAMP", [2.5]) is None and _fn("VAR_POP", [2.5]) == 0.0 and _fn("VAR_POP", []) is None
    assert _fn("VAR_SAMP", [1.0, 3.0]) == 2.0 and _fn("STDDEV_POP", [1.0, 3.0]) == 1.0
    assert _fn("VAR_SAMP", [7.0] * 9) == 0.0
    for bad in (math.nan, math.inf, -math.inf):
        assert math.isnan(_fn("VAR_POP", [1.0, bad, 2.0]))
    r = OM.running_moments([1.0, None, 3.0, math.inf])
    assert r[:3] == [(1, 0.0), (1, 0.0), (2, 2.0)] and math.isnan(r[3][1])
    assert OM.running_moments([None]) == [(0, None)]


def test_dyadic_sums_agree_with_fractions():
    rng = np.random.default_rng(2)
    n = 5000
    g = rng.integers(0, 40, n)
    k = rng.integers(-(1 << 20) + 1, 1 << 20, n)
    valid = rng.random(n) > 0.1
    fast = OM.dyadic_group_moments(g, k, valid)
    slow = OM.group_moments(g.tolist(), [x / 1024 if ok else None for x, ok in zip(k.tolist(), valid)])
    assert fast == {key: mv for key, mv in slow.items() if mv[0] > 0}
