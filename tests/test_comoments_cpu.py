"""CORR / COVAR_* / REGR_* without a GPU: builders, types and names, SQL, rejections, the K6 accumulator plan, the
exact reference against statistics / numpy / pandas, and a model of why the textbook formula is not used."""
import math
import statistics
import types
from fractions import Fraction

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

from fugue_b200 import kernels as K
from fugue_b200.column import BIVARIATES, Kind, SelectColumns, col, functions as f, to_sql
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.dist import DistributedB200Engine
from fugue_b200.execution_engine import B200ExecutionEngine, decompose_aggs
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select
from fugue_b200.table import B200Table
from oracle import comoments as OC

FUNCS = sorted(BIVARIATES)


def build(fn, a, b):
    return getattr(f, fn.lower())(a, b)


# ---- IR ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", FUNCS)
def test_builders_types_and_names(fn):
    e = build(fn, col("a"), "b")
    assert e.kind == Kind.AGG and e.func == fn and [x.name for x in e.args] == ["a", "b"] and not e.is_distinct
    assert e.fingerprint() == build(fn, "a", "b").fingerprint()
    assert e.infer_alias().output_name == ""  # two arguments: no implicit name
    assert e.alias("r").infer_alias().output_name == "r"
    schema = Schema("a:int,b:double")
    assert e.infer_type(schema) == (pa.int64() if fn == "REGR_COUNT" else pa.float64())
    w = e.over()
    assert w.kind == Kind.WINDOW and w.args == e.args and w.infer_type(schema) == e.infer_type(schema)
    assert e.over(running=True).kwargs == {"running": True}
    assert f.is_agg(e) and f.is_agg(e * 2 + 1) and not f.is_agg(w)
    with pytest.raises(ValueError):
        build(fn, col("*"), "b")
    with pytest.raises(ValueError):
        build(fn, f.sum(col("a")), "b")


def test_x_and_y_of_the_pair():
    from fugue_b200.column import bivariate_xy

    assert [e.name for e in bivariate_xy(f.corr("a", "b"))] == ["a", "b"]
    assert [e.name for e in bivariate_xy(f.regr_slope("y", "x"))] == ["x", "y"]  # REGR_*(y, x)


@pytest.mark.parametrize("kw", [{"rows": (-2, 0)}, {"rows": (0, 3)}, {"range": (-1.0, 0)}, {"range": (None, 0)}])
def test_frames_are_not_supported(kw):
    for fn in FUNCS:
        with pytest.raises(NotImplementedError, match="ROWS and RANGE frames are not supported"):
            build(fn, "a", "b").over(**kw)


# ---- SQL ---------------------------------------------------------------------------------------------
def _parse(items, rest="FROM t"):
    return _parse_select(items, rest, f"SELECT {items} {rest}")


@pytest.mark.parametrize("fn", FUNCS)
def test_sql_names_and_print_parse_fixed_point(fn):
    e = build(fn, col("y"), col("x") * 2).alias("r")
    text = to_sql(e)
    assert text == f"{fn}(y,x*2) AS r"
    (back,) = _parse(text).columns
    assert back.fingerprint() == e.fingerprint() and to_sql(back) == text
    (low,) = _parse(f"{fn.lower()}(y, x * 2) AS r").columns
    assert low.fingerprint() == e.fingerprint()


def test_regr_argument_order_survives_sql():
    (e,) = _parse("REGR_SLOPE(dep, indep) AS s").columns
    assert [a.name for a in e.args] == ["dep", "indep"]
    from fugue_b200.column import bivariate_xy

    assert [a.name for a in bivariate_xy(e)] == ["indep", "dep"]


def test_sql_rejects_distinct_and_one_argument():
    for fn in FUNCS:
        with pytest.raises(NotImplementedError, match="DISTINCT"):
            _parse(f"{fn}(DISTINCT a, b) AS r")
        with pytest.raises(NotImplementedError):
            _parse(f"{fn}(a) AS r")


# ---- rejections before any device work ---------------------------------------------------------------
def test_no_partial_final_form_and_multi_gpu_raises():
    for fn in FUNCS:
        with pytest.raises(NotImplementedError):
            decompose_aggs([build(fn, col("a"), col("b")).alias("r")])
    t = B200Table(Schema("k:long,a:double,b:double"), [torch.tensor([1, 2]), torch.tensor([1.0, 2.0]),
                                                          torch.tensor([3.0, 1.0])])
    fake = types.SimpleNamespace(_world=2, to_df=lambda df: df, _plain_aggs=B200ExecutionEngine._plain_aggs)
    for fn in FUNCS:
        for spec in (PartitionSpec(by=["k"]), None):
            with pytest.raises(NotImplementedError):
                DistributedB200Engine.aggregate(fake, B200DataFrame(t), spec, [build(fn, col("a"), col("b")).alias("r")])


def test_plain_aggs_take_named_pairs_only():
    assert B200ExecutionEngine._plain_aggs([build(fn, col("a"), col("b")).alias("r") for fn in FUNCS])
    assert not B200ExecutionEngine._plain_aggs([f.corr(col("a") + 1, col("b")).alias("r")])
    assert not B200ExecutionEngine._plain_aggs([f.corr(col("a"), col("b").cast("int")).alias("r")])


def test_count_distinct_in_the_same_select_raises_before_device_work(monkeypatch):
    import fugue_b200.expr as X

    def no_device(*a, **k):
        raise AssertionError("device work before the rejection")

    monkeypatch.setattr(X, "project", no_device)
    t = B200Table(Schema("k:long,a:double,b:double"), [torch.tensor([1]), torch.tensor([1.0]), torch.tensor([2.0])])
    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)
    eng.to_df = lambda df: df
    sel = SelectColumns(col("k"), f.corr(col("a"), col("b")).alias("c"), f.count_distinct(col("a")).alias("n"))
    with pytest.raises(NotImplementedError, match="COUNT\\(DISTINCT"):
        B200ExecutionEngine.select(eng, B200DataFrame(t), sel)


@pytest.mark.parametrize("tp", ["str", "bool", "date", "datetime"])
def test_non_numeric_arguments_raise(tp):
    store = {"str": torch.tensor([0, 1], dtype=torch.int32), "bool": torch.tensor([1, 0], dtype=torch.uint8),
             "date": torch.tensor([0, 1], dtype=torch.int32), "datetime": torch.tensor([0, 1])}[tp]
    t = B200Table(Schema(f"k:long,v:double,s:{tp}"), [torch.tensor([1, 2]), torch.tensor([1.0, 2.0]), store],
                  [None] * 3, {"s": pa.array(["a", "b"])} if tp == "str" else {})
    add = lambda *a: 0  # noqa: E731
    with pytest.raises(NotImplementedError):
        B200ExecutionEngine._pair_accumulators(t, f.corr("s", "v"), ("s", "v"), add, {}, {})


# ---- the K6 accumulator plan -------------------------------------------------------------------------
def _cpu_table(tbl: pa.Table) -> B200Table:
    """A host-memory table of int / float columns (NULL: a validity byte of 0)."""
    cols, valid = [], []
    for c in tbl.columns:
        a = c.combine_chunks()
        cols.append(torch.from_numpy(a.fill_null(0).to_numpy(zero_copy_only=False).copy()))
        valid.append(None if a.null_count == 0 else torch.from_numpy(a.is_valid().to_numpy(zero_copy_only=False)
                                                                     .astype(np.uint8)))
    return B200Table(Schema(tbl.schema), cols, valid)


def _plan(tbl: pa.Table, aggs):
    """The accumulators ``_aggregate_named`` asks K6 for, captured instead of launched."""
    t = _cpu_table(tbl)
    seen = {}

    def fake_groupby(key64, kvalid, vals, vvalid, ops):
        seen.update(vals=vals, valid=vvalid, ops=ops)
        raise StopIteration

    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)
    eng.to_df = lambda df: df
    sorted_calls = []
    eng._aggregate_sorted = lambda df, spec, a: sorted_calls.append(a) or "sorted"
    old = K.groupby_u64
    K.groupby_u64 = fake_groupby
    try:
        try:
            r = B200ExecutionEngine._aggregate_named(eng, B200DataFrame(t), PartitionSpec(by=["k"]), aggs)
        except StopIteration:
            r = None
    finally:
        K.groupby_u64 = old
    return r, seen, sorted_calls


def test_k6_plan_is_12_accumulators_shared_by_the_pair():
    tbl = pa.table({"k": [1, 1, 2], "x": pa.array([1.0, None, 3.0]), "y": pa.array([2, 5, None], pa.int32())})
    aggs = [build(fn, col("y"), col("x")).alias(fn) if fn.startswith("REGR_") else build(fn, col("x"), col("y")).alias(fn)
            for fn in FUNCS]
    r, seen, srt = _plan(tbl, aggs)
    assert r is None and not srt
    ops = seen["ops"]
    assert len(ops) == 12  # every function of the pair (x, y) shares one set
    assert ops == [K.AGG_SUM_F64, K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64, K.AGG_CODEV_F64,
                   K.AGG_DEV_F64, K.AGG_DEV2_F64, K.AGG_MIN_F64, K.AGG_MAX_F64, K.AGG_MIN_F64, K.AGG_MAX_F64]
    pv = seen["valid"][0]
    assert all(v is pv for v in seen["valid"])  # ONE pair validity tensor
    assert pv.tolist() == [1, 0, 0]  # x valid AND y valid
    x, y = seen["vals"][0], seen["vals"][1]
    assert seen["vals"][5] is x and seen["vals"][6] is y  # CODEV names x, the DEV after it y
    assert x.dtype == y.dtype == torch.float64


def test_k6_plan_single_side_mask_and_same_column_twice():
    tbl = pa.table({"k": [1, 2], "x": pa.array([1.0, None]), "y": [2.0, 3.0]})
    _, seen, _ = _plan(tbl, [f.corr(col("x"), col("y")).alias("c")])
    assert all(v is seen["valid"][0] for v in seen["valid"]) and seen["valid"][0].tolist() == [1, 0]
    _, seen, _ = _plan(pa.table({"k": [1, 2], "x": [1.0, 2.0]}), [f.corr(col("x"), col("x")).alias("c")])
    assert all(v is None for v in seen["valid"])
    ops = seen["ops"]
    assert len(ops) == 10 and ops.count(K.AGG_SUM_F64) == 1 and ops.count(K.AGG_DEV_F64) == 2  # x's set, and the
    c = ops.index(K.AGG_CODEV_F64)                                                            # DEV tied to the CODEV
    assert ops[c + 1] == K.AGG_DEV_F64 and seen["vals"][c + 1] is seen["vals"][c]


@pytest.mark.parametrize("pair_first", [False, True])
@pytest.mark.parametrize("xnull", [False, True])
def test_k6_plan_shares_deviation_sets_with_variances(pair_first, xnull):
    """CORR(x, y) beside STDDEV(x) and VAR_POP(y): one (SUM, COUNT, DEV, DEV2) set per (column, validity), so K6
    never sees two DEVs of the same column (it would give each its own sums, but the sets would be spent twice)."""
    tbl = pa.table({"k": [1, 1, 2], "x": pa.array([1.0, None if xnull else 2.0, 3.0]), "y": [2.0, 5.0, 4.0]})
    pair, var = [f.corr(col("x"), col("y")).alias("r")], [f.stddev(col("x")).alias("s"), f.var_pop(col("y")).alias("v")]
    _, seen, srt = _plan(tbl, pair + var if pair_first else var + pair)
    assert not srt
    ops, vals, valid = seen["ops"], seen["vals"], seen["valid"]
    sums = [(vals[i].data_ptr(), None if valid[i] is None else valid[i].data_ptr())
            for i, o in enumerate(ops) if o == K.AGG_SUM_F64]
    assert len(sums) == len(set(sums))  # one set per (column, validity)
    # STDDEV(x) shares the pair's x set (the pair validity is x's own mask, or none).  VAR_POP(y) has y's own
    # validity (none): it shares the pair's y set when the pair validity is none too, and when it came first the
    # pair adds only the DEV of y tied to its CODEV
    assert len(ops) == {(True, False): 12, (False, False): 14}.get((pair_first, xnull), 16)
    c = ops.index(K.AGG_CODEV_F64)
    assert ops[c + 1] == K.AGG_DEV_F64 and valid[c + 1] is valid[c]


def test_k6_plan_past_16_takes_the_sorted_route():
    tbl = pa.table({"k": [1], "a": [1.0], "b": [2.0], "c": [3.0]})
    r, seen, srt = _plan(tbl, [f.corr(col("a"), col("b")).alias("p"), f.corr(col("a"), col("c")).alias("q")])
    assert r == "sorted" and len(srt) == 1 and not seen
    r, seen, srt = _plan(tbl, [f.corr(col("a"), col("b")).alias("p"), f.stddev(col("c")).alias("s")])
    assert r is None and len(seen["ops"]) == 16 and not srt
    # without the family, past 16 still raises as before
    many = [f.stddev(col(c)).alias(f"s{c}") for c in "abc"] + [f.sum(col(c)).alias(f"t{c}") for c in "abc"] + \
        [f.min(col(c)).alias(f"u{c}") for c in "abc"]
    with pytest.raises(NotImplementedError, match="accumulators"):
        _plan(tbl, many)


# ---- the oracle against independent references ---------------------------------------------------------
def _data(seed, n=60):
    rng = np.random.default_rng(seed)
    x = rng.normal(3, 2, n)
    y = x * rng.normal(0.4, 0.2) + rng.normal(0, 1, n)
    return x.tolist(), y.tolist()


@pytest.mark.parametrize("seed", range(5))
def test_oracle_against_statistics(seed):
    x, y = _data(seed)
    assert OC.result_exact("COVAR_SAMP", x, y) == pytest.approx(statistics.covariance(x, y), rel=1e-13)
    assert OC.result_exact("CORR", x, y) == pytest.approx(statistics.correlation(x, y), rel=1e-13)
    lr = statistics.linear_regression(x, y)
    assert OC.result_exact("REGR_SLOPE", x, y) == pytest.approx(lr.slope, rel=1e-13)
    assert OC.result_exact("REGR_INTERCEPT", x, y) == pytest.approx(lr.intercept, rel=1e-12)
    assert OC.result_exact("REGR_AVGX", x, y) == pytest.approx(statistics.fmean(x), rel=1e-15)
    assert OC.result_exact("REGR_R2", x, y) == pytest.approx(statistics.correlation(x, y) ** 2, rel=1e-13)


@pytest.mark.parametrize("seed", range(5))
def test_oracle_against_numpy(seed):
    x, y = _data(seed)
    c = np.cov(x, y)
    assert OC.result_exact("COVAR_SAMP", x, y) == pytest.approx(c[0, 1], rel=1e-13)
    assert OC.result_exact("COVAR_POP", x, y) == pytest.approx(np.cov(x, y, ddof=0)[0, 1], rel=1e-13)
    assert OC.result_exact("CORR", x, y) == pytest.approx(np.corrcoef(x, y)[0, 1], rel=1e-13)
    slope, icept = np.polyfit(x, y, 1)
    assert OC.result_exact("REGR_SLOPE", x, y) == pytest.approx(slope, rel=1e-12)
    assert OC.result_exact("REGR_INTERCEPT", x, y) == pytest.approx(icept, rel=1e-11)
    n = len(x)
    assert OC.result_exact("REGR_SXX", x, y) == pytest.approx(c[0, 0] * (n - 1), rel=1e-13)
    assert OC.result_exact("REGR_SYY", x, y) == pytest.approx(c[1, 1] * (n - 1), rel=1e-13)
    assert OC.result_exact("REGR_SXY", x, y) == pytest.approx(c[0, 1] * (n - 1), rel=1e-13)


def test_oracle_grouped_against_pandas():
    rng = np.random.default_rng(7)
    n = 3000
    pdf = pd.DataFrame({"k": rng.integers(0, 20, n), "x": rng.normal(0, 5, n)})
    pdf["y"] = pdf["x"] * 0.2 + rng.normal(1, 1, n)
    pdf.loc[rng.random(n) < 0.1, "x"] = np.nan  # NULL in the NaN-free sense: pandas drops the row, so do we
    xs = [None if math.isnan(v) else v for v in pdf["x"]]
    st = OC.group_states(pdf["k"].tolist(), xs, pdf["y"].tolist())
    g = pdf.groupby("k")
    cov = g.apply(lambda d: d["x"].cov(d["y"]))
    cor = g.apply(lambda d: d["x"].corr(d["y"]))
    for k, s in st.items():
        assert OC.result_of_state("COVAR_SAMP", s) == pytest.approx(cov[k], rel=1e-12)
        assert OC.result_of_state("CORR", s) == pytest.approx(cor[k], rel=1e-12)


def test_oracle_null_nan_and_clamp_rules():
    assert OC.result_exact("REGR_COUNT", [None, 1.0], [2.0, None]) == 0
    for fn in FUNCS:
        if fn != "REGR_COUNT":
            assert OC.result_exact(fn, [None], [1.0]) is None
    assert OC.result_exact("COVAR_SAMP", [1.0], [2.0]) is None and OC.result_exact("COVAR_POP", [1.0], [2.0]) == 0.0
    const = [0.1] * 5
    assert OC.result_exact("CORR", const, [1, 2, 3, 4, 5]) is None
    assert OC.result_exact("REGR_SLOPE", const, [1, 2, 3, 4, 5]) is None
    assert OC.result_exact("REGR_SXY", const, [1, 2, 3, 4, 5]) == 0.0
    assert OC.result_exact("REGR_R2", [1, 2, 3], const[:3]) == 1.0
    assert OC.result_exact("CORR", [1, 2, 3], const[:3]) is None
    assert math.isnan(OC.result_exact("CORR", [1.0, math.nan, 2.0], [1.0, 2.0, 4.0]))
    assert math.isnan(OC.result_exact("REGR_SYY", [1.0, math.inf], [1.0, 2.0]))  # inf in x poisons Syy too
    assert OC.result_exact("REGR_AVGY", [1.0, 2.0], [math.inf, 2.0]) == math.inf
    assert math.isnan(OC.result_exact("REGR_AVGX", [-math.inf, math.inf], [1.0, 2.0]))
    assert OC.result_exact("CORR", [1.0, 2.0, 3.0], [2.0, 4.0, 6.0]) == 1.0
    assert OC.result_exact("CORR", [1.0, 2.0, 3.0], [3.0, 2.0, 1.0]) == -1.0


def test_running_and_dyadic_forms_agree_with_the_direct_one():
    rng = np.random.default_rng(3)
    n = 400
    kx, ky = rng.integers(-1000, 1000, n), rng.integers(-1000, 1000, n)
    valid = rng.random(n) > 0.2
    xs = [v / 1024 if ok else None for v, ok in zip(kx.tolist(), valid)]
    ys = (ky / 1024).tolist()
    run = OC.running_states(xs, ys)
    for i in (0, 10, 199, n - 1):
        assert run[i] == OC.exact_state(OC.pair_rows(xs[:i + 1], ys[:i + 1]))
    gid = np.arange(n) % 3
    dy = OC.dyadic_group_states(gid, kx, ky, valid)
    for g in range(3):
        sel = gid == g
        want = OC.exact_state(OC.pair_rows([x for x, s in zip(xs, sel) if s], [y for y, s in zip(ys, sel) if s]))
        assert dy[g] == want


# ---- why the textbook formula is not used ---------------------------------------------------------------
def test_textbook_formula_fails_on_shifted_data_where_the_corrected_one_passes():
    """Means 1e9, sigma 1e-3: sum xy - sum x sum y / m in float64 misses the K6 bound of
    tests/test_comoments_gpu.py by orders of magnitude; the corrected two-pass (modelled in numpy with the
    device's operation order: mean from the sums, then CODEV - DEVx DEVy / m) meets it."""
    rng = np.random.default_rng(1)
    u = 2.0 ** -53
    fails_textbook = fails_corrected = 0
    for _ in range(20):
        m = 500
        x = 1e9 + rng.standard_normal(m) * 1e-3
        y = 1e9 + (x - 1e9) * 0.5 + rng.standard_normal(m) * 1e-3
        _, _, _, sxx, syy, sxy = OC.exact_state(list(zip(x.tolist(), y.tolist())))
        nx, ny = math.sqrt(float(sum(Fraction(v) ** 2 for v in x))), math.sqrt(float(sum(Fraction(v) ** 2 for v in y)))
        bound = 2 * ((m + 2) * u * math.sqrt(float(sxx) * float(syy)) + (m * u) ** 2 * nx * ny)
        textbook = float(np.sum(x * y) - np.sum(x) * np.sum(y) / m)
        mx, my = np.sum(x) / m, np.sum(y) / m
        dx, dy = x - mx, y - my
        corrected = float(np.sum(dx * dy) - np.sum(dx) * np.sum(dy) / m)
        fails_textbook += abs(textbook - float(sxy)) > bound
        fails_corrected += abs(corrected - float(sxy)) > bound
    assert fails_textbook == 20 and fails_corrected == 0
