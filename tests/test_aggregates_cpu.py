"""The per-function semantics of ``fugue_b200/aggregates.py`` on host tensors, at the edge states both routes meet
(count 0, count 1, a constant column, NaN and +-inf, no validity), and the catalogue of aggregate heads in
``column.AGGREGATES`` against the builders and ``over()``."""
import math

import pyarrow as pa
import pytest
import torch

from fugue_b200 import aggregates as A
from fugue_b200 import kernels as K
from fugue_b200.column import AGGREGATES, BIVARIATES, ColumnExpr, Kind, col, functions as f
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table

NAN, INF = math.nan, math.inf


def i64(*v):
    return torch.tensor(v, dtype=torch.int64)


def f64(*v):
    return torch.tensor(v, dtype=torch.float64)


def same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Equal dtype and bits (NaN included)."""
    return a.dtype == b.dtype and a.shape == b.shape and bool((a.view(torch.uint8) == b.view(torch.uint8)).all())


# ---- reduce_input ------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn,tp,store,op,dtype", [
    ("SUM", pa.int32(), torch.int32, K.AGG_SUM_I64, torch.int64),
    ("SUM", pa.float32(), torch.float32, K.AGG_SUM_F64, torch.float64),
    ("AVG", pa.int32(), torch.int32, K.AGG_SUM_F64, torch.float64),
    ("AVG", pa.float64(), torch.float64, K.AGG_SUM_F64, torch.float64),
    ("MIN", pa.uint32(), torch.int32, K.AGG_MIN_I64, torch.int64),
    ("MAX", pa.float64(), torch.float64, K.AGG_MAX_F64, torch.float64),
    ("MIN", pa.date32(), torch.int32, K.AGG_MIN_I64, torch.int64),
    ("FIRST", pa.int64(), torch.int64, K.AGG_MIN_I64, torch.int64),
    ("LAST", pa.int64(), torch.int64, K.AGG_MAX_I64, torch.int64)])
def test_reduce_input_op_and_values(fn, tp, store, op, dtype):
    c = torch.tensor([3, -1, 7], dtype=store)
    got_op, v = A.reduce_input(fn, c, tp)
    assert got_op == op and v.dtype == dtype and v.is_contiguous()
    want = c.to(torch.int64) & 0xFFFFFFFF if tp == pa.uint32() else c.to(dtype)
    assert torch.equal(v, want)
    if c.dtype == dtype:  # an 8-byte column of the right class is passed as it is: K6 ties columns by pointer
        assert v is c


def test_f64_values_cache_keeps_one_tensor_per_column():
    t = B200Table(Schema("a:int,b:double"), [torch.tensor([1, 2], dtype=torch.int32), f64(0.5, NAN)])
    cache = {}
    a = A.f64_values(t, "a", cache)
    assert a.dtype == torch.float64 and a.tolist() == [1.0, 2.0]
    assert A.f64_values(t, "a", cache) is a
    assert A.f64_values(t, "a") is not a  # without a cache, a fresh widening
    assert A.f64_values(t, "b", cache) is t.columns[1]


# ---- check_argument ----------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", ["VAR_SAMP", "STDDEV_POP", "CORR", "REGR_COUNT"])
@pytest.mark.parametrize("tp,is_dict", [(pa.string(), True), (pa.bool_(), False), (pa.date32(), False),
                                        (pa.timestamp("us"), False)])
def test_numeric_only_functions_reject(fn, tp, is_dict):
    with pytest.raises(NotImplementedError):
        A.check_argument(fn, "a", tp, is_dict)


@pytest.mark.parametrize("fn", ["VAR_POP", "COVAR_SAMP", "SUM", "AVG", "MIN", "MAX", "COUNT", "FIRST", "LAST"])
@pytest.mark.parametrize("tp", [pa.int8(), pa.uint64(), pa.float16(), pa.float64()])
def test_numeric_arguments_pass(fn, tp):
    A.check_argument(fn, "a", tp, False)


def test_strings_take_min_max_count_and_picks_only():
    for fn in ("MIN", "MAX", "COUNT", "FIRST", "LAST"):
        A.check_argument(fn, "s", pa.string(), True)
    for fn in ("SUM", "AVG"):
        with pytest.raises(NotImplementedError):
            A.check_argument(fn, "s", pa.string(), True)
    A.check_argument("SUM", "d", pa.date32(), False)  # other non-numeric columns reduce as their storage


# ---- finish_basic ------------------------------------------------------------------------------------
def test_count_is_never_null():
    c, v, tp = A.finish_basic("COUNT", None, i64(0, 1, 5), None)
    assert c.tolist() == [0, 1, 5] and v is None and tp == pa.int64()


@pytest.mark.parametrize("fn,arg,value,out", [
    ("SUM", pa.int32(), i64(0, -7, 9), pa.int64()),
    ("SUM", pa.float32(), f64(0.0, 2.5, -INF), pa.float64()),
    ("MIN", pa.int16(), i64(0, -7, 9), pa.int16()),
    ("MAX", pa.float32(), f64(0.0, INF, NAN), pa.float32()),
    ("MIN", pa.date32(), i64(0, 18000, 3), pa.date32()),
    ("MAX", pa.float16(), f64(0.0, 0.5, -2.0), pa.float16())])
def test_sum_min_max_are_null_at_count_0(fn, arg, value, out):
    count = i64(0, 1, 3)
    c, v, tp = A.finish_basic(fn, value, count, arg)
    assert tp == out and v.tolist() == [0, 1, 1] and c.is_contiguous()
    back = c.view(torch.float16).to(torch.float64) if out == pa.float16() else c.to(value.dtype)
    assert same(back, value)
    c2, v2, _ = A.finish_basic(fn, value, None, arg)  # a keyed aggregate of a column without NULLs
    assert v2 is None and same(c2, c)


def test_avg_divides_by_the_count():
    c, v, tp = A.finish_basic("AVG", f64(0.0, 3.0, 6.0, INF, NAN), i64(0, 1, 3, 2, 2), pa.int64())
    assert tp == pa.float64() and v.tolist() == [0, 1, 1, 1, 1]
    assert c.tolist()[1:3] == [3.0, 2.0] and c[3].item() == INF and math.isnan(c[4].item())
    assert A.divides_by_count("AVG") and not any(A.divides_by_count(fn) for fn in ("SUM", "MIN", "MAX", "COUNT"))


def test_min_equals_max_on_a_constant_column():
    mn = A.finish_basic("MIN", f64(0.1, 0.1), i64(4, 1), pa.float64())
    mx = A.finish_basic("MAX", f64(0.1, 0.1), i64(4, 1), pa.float64())
    assert same(mn[0], mx[0]) and mn[1].tolist() == mx[1].tolist() == [1, 1]


def test_string_min_max_map_ranks_back_to_codes():
    d = pa.array(["b", "a", "c"])  # ranks in code-point order: a 0, b 1, c 2
    c, v, tp, dd = A.finish_string(i64(0, 2, 1, 0), i64(1, 2, 5, 0), d, pa.string())
    assert c.dtype == torch.int32 and [d[i].as_py() for i in c.tolist()[:3]] == ["a", "c", "b"]
    assert v.tolist() == [1, 1, 1, 0] and tp == pa.string() and dd is d


# ---- variances -------------------------------------------------------------------------------------
def test_m2_is_clamped_at_zero():
    assert A.m2_of(f64(1.0, 0.0, 1.0), f64(0.4, 2.0, 0.5), f64(2.0, 2.0, 2.0)).tolist() == [0.0, 2.0, 0.0]


@pytest.mark.parametrize("fn,want", [("VAR_SAMP", [None, None, 8 / 3, 0.0]), ("VAR_POP", [None, 0.0, 2.0, 0.0]),
                                     ("STDDEV_SAMP", [None, None, math.sqrt(8 / 3), 0.0]),
                                     ("STDDEV_POP", [None, 0.0, math.sqrt(2.0), 0.0])])
def test_variance_null_rules(fn, want):
    v, ok = A.variance_of(fn, f64(0.0, 0.0, 8.0, 0.0), i64(0, 1, 4, 5))  # count 0, count 1, spread, constant
    assert [x if o else None for x, o in zip(v.tolist(), ok.tolist())] == pytest.approx(want, rel=1e-15)
    nan, _ = A.variance_of(fn, f64(NAN), i64(3))
    assert math.isnan(nan.item())


# ---- two-argument functions --------------------------------------------------------------------------
def _moments(m, mx, my, sxx, syy, sxy):
    return [i64(m)] + [f64(v) for v in (mx, my, sxx, syy, sxy)]


def _biv(fn, *st):
    v, ok = A.bivariate_of(fn, *_moments(*st))
    return v.item() if ok is None or ok.item() else None


def test_bivariates_at_count_0_and_1():
    for fn in sorted(BIVARIATES):
        assert _biv(fn, 0, 0.0, 0.0, 0.0, 0.0, 0.0) == (0 if fn == "REGR_COUNT" else None)
    assert _biv("REGR_COUNT", 1, 2.0, 3.0, 0.0, 0.0, 0.0) == 1
    assert _biv("COVAR_SAMP", 1, 2.0, 3.0, 0.0, 0.0, 0.0) is None
    assert _biv("COVAR_POP", 1, 2.0, 3.0, 0.0, 0.0, 0.0) == 0.0
    assert _biv("REGR_AVGX", 1, 2.0, 3.0, 0.0, 0.0, 0.0) == 2.0
    assert _biv("CORR", 1, 2.0, 3.0, 0.0, 0.0, 0.0) is None


def test_bivariates_of_constant_columns():
    # constant x: Sxx = Sxy = 0
    for fn in ("CORR", "REGR_SLOPE", "REGR_INTERCEPT", "REGR_R2"):
        assert _biv(fn, 4, 0.1, 1.0, 0.0, 5.0, 0.0) is None
    assert _biv("REGR_SXX", 4, 0.1, 1.0, 0.0, 5.0, 0.0) == 0.0
    # constant y: CORR NULL, R2 1, slope 0
    assert _biv("CORR", 4, 1.0, 0.1, 5.0, 0.0, 0.0) is None
    assert _biv("REGR_R2", 4, 1.0, 0.1, 5.0, 0.0, 0.0) == 1.0
    assert _biv("REGR_SLOPE", 4, 1.0, 0.1, 5.0, 0.0, 0.0) == 0.0


def test_bivariates_clamp_and_propagate_nan():
    assert _biv("CORR", 3, 0.0, 0.0, 1.0, 1.0, 1.0 + 1e-15) == 1.0
    assert _biv("REGR_R2", 3, 0.0, 0.0, 1.0, 1.0, 1.0 + 1e-15) == 1.0
    for fn in ("CORR", "REGR_SLOPE", "REGR_R2", "COVAR_POP"):
        assert math.isnan(_biv(fn, 3, 0.0, 0.0, NAN, NAN, NAN))


def _bits(*v):
    return f64(*v).view(torch.int64)


def _pair_gaggs(x, y):
    """The 12 accumulators of a pair over rows (x, y) as K6 leaves them: deviations from the mean."""
    m = len(x)
    mx, my = sum(x) / m, sum(y) / m
    dx, dy = [a - mx for a in x], [b - my for b in y]
    return [_bits(sum(x)), _bits(sum(y)), i64(m), _bits(sum(dx)), _bits(sum(a * a for a in dx)),
            _bits(sum(a * b for a, b in zip(dx, dy))), _bits(sum(dy)), _bits(sum(b * b for b in dy)),
            _bits(min(x)), _bits(max(x)), _bits(min(y)), _bits(max(y))]


def test_pair_moments_constant_and_finite_rules():
    slots = tuple(range(12))
    m, mx, my, sxx, syy, sxy = (v.item() for v in A.pair_moments(_pair_gaggs([1.0, 3.0], [2.0, 2.0]), slots))
    assert (m, mx, my, sxx, syy, sxy) == (2, 2.0, 2.0, 2.0, 0.0, 0.0)
    g = _pair_gaggs([1.0, 3.0], [2.0, 5.0])
    g[9] = _bits(INF)  # an infinite MAX of x: every S is NaN
    st = A.pair_moments(g, slots)
    assert all(math.isnan(v.item()) for v in st[3:])


# ---- the catalogue -----------------------------------------------------------------------------------
def _built_aggregates():
    """Every AGG head a builder of ``column.functions`` produces."""
    heads = set()
    for name in dir(f):
        b = getattr(f, name)
        if name.startswith("_") or not callable(b):
            continue
        for args in ((col("a"),), (col("a"), col("b")), (col("a"), 0.5)):
            try:
                e = b(*args)
            except Exception:  # noqa: BLE001 - builders of other arities or argument kinds
                continue
            if isinstance(e, ColumnExpr) and e.kind == Kind.AGG:
                heads.add(e.head)
    return heads


def test_every_built_aggregate_has_an_entry():
    heads = _built_aggregates()
    assert {"SUM", "COUNT", "AVG", "MIN", "MAX", "FIRST", "LAST", "PERCENTILE_CONT", "STDDEV_SAMP", "CORR",
            "REGR_R2"} <= heads
    assert heads <= set(AGGREGATES)


def _node(head):
    a = AGGREGATES[head]
    args = [col("a"), col("b")] if a.family == "bivariate" else [col("a")]
    return ColumnExpr(Kind.AGG, head, args, {"q": 0.5} if a.family == "percentile" else None)


@pytest.mark.parametrize("head", sorted(AGGREGATES))
def test_frame_rule_is_what_over_accepts(head):
    frames = AGGREGATES[head].frames
    e = _node(head)
    assert e.over().kind == Kind.WINDOW
    for kw in ({"running": True}, {"rows": (-2, 1)}, {"range": (-1, 1)}):
        if frames == "any" or (frames == "running" and "running" in kw):
            assert e.over(**kw).kind == Kind.WINDOW
        else:
            with pytest.raises(NotImplementedError if frames == "running" else ValueError):
                e.over(**kw)


def test_heads_outside_the_catalogue_have_no_window_form():
    with pytest.raises(ValueError, match="no window form"):
        ColumnExpr(Kind.AGG, "MODE", [col("a")]).over()
