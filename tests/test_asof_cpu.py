"""As-of joins on the CPU (DESIGN §7q): the oracle against ``pandas.merge_asof``, its NULL / NaN / key rules on
hand-written rows, the schema rule, the tolerance rules, the SQL forms parsed to the engine call, and every
rejection, all before any device work."""
import datetime
import math

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from fugue_b200 import kernels as K
from fugue_b200.join import asof_key_class, asof_tolerance, get_asof_schemas
from fugue_b200.schema import Schema, SchemaError
from oracle import asof as A


def _pandas_rows(left: pd.DataFrame, right: pd.DataFrame, by, direction, exact, tol):
    res = pd.merge_asof(left, right, on="t", by=by or None, direction=direction, allow_exact_matches=exact,
                        tolerance=tol)
    return [-1 if (isinstance(v, float) and math.isnan(v)) else int(v) for v in res["rid"]]


@pytest.mark.parametrize("nkeys", [0, 1, 2])
@pytest.mark.parametrize("direction", A.DIRECTIONS)
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("tol", [None, 0, 3])
def test_oracle_equals_merge_asof(nkeys, direction, exact, tol):
    rng = np.random.default_rng(nkeys * 100 + len(direction) * 10 + exact + (tol or 0))
    n1, n2 = 400, 300
    right = pd.DataFrame({"t": np.sort(rng.integers(0, 200, n2)), "rid": np.arange(n2)})
    left = pd.DataFrame({"t": np.sort(rng.integers(-5, 210, n1))})
    by = [f"k{i}" for i in range(nkeys)]
    for k in by:
        right[k] = rng.integers(0, 4, n2)
        left[k] = rng.integers(0, 5, n1)  # key 4 has no right rows
    got = A.match_rows(list(zip(*[left[k].tolist() for k in by])) or [()] * n1, left["t"].tolist(),
                       list(zip(*[right[k].tolist() for k in by])) or [()] * n2, right["t"].tolist(), direction, exact,
                       tol)
    assert got == _pandas_rows(left, right, by, direction, exact, tol)
    lk = (left[by[0]].to_numpy() if nkeys else np.zeros(n1, np.int64)).astype(np.int64)
    rk = (right[by[0]].to_numpy() if nkeys else np.zeros(n2, np.int64)).astype(np.int64)
    if nkeys == 2:  # one int64 surrogate of the pair
        lk, rk = lk * 8 + left["k1"].to_numpy(), rk * 8 + right["k1"].to_numpy()
    fast = A.match_rows_np(lk, left["t"].to_numpy(np.int64), np.ones(n1, bool), rk, right["t"].to_numpy(np.int64),
                           np.ones(n2, bool), direction, exact, tol)
    assert fast.tolist() == got


@pytest.mark.parametrize("direction,expect", [("backward", [1, 1, 3]), ("forward", [2, 2, 4]),
                                              ("nearest", [1, 1, 4])])
def test_ties(direction, expect):
    """Right t = [3, 3, 7, 7, 12] carrying rows [a, b, c, d, e], left t = [5, 5, 10]: backward takes the last of
    equal values, forward the first, nearest the backward one on equal distance."""
    rt, lt = [3, 3, 7, 7, 12], [5, 5, 10]
    assert A.match_rows([()] * 3, lt, [()] * 5, rt, direction) == expect
    assert _pandas_rows(pd.DataFrame({"t": lt}), pd.DataFrame({"t": rt, "rid": range(5)}), [], direction, True,
                        None) == expect


def test_nearest_strict_ties():
    assert A.match_rows([()] * 2, [5, 7], [()] * 4, [3, 5, 7, 9], "nearest", False) == [0, 1]
    assert A.match_rows([()] * 2, [5, 7], [()] * 4, [3, 5, 7, 9], "nearest", True) == [1, 2]


def test_oracle_null_nan_and_key_rules():
    left = pa.table({"k": pa.array([1.0, None, float("nan"), -0.0, 2.0, 2.0], pa.float64()),
                     "t": pa.array([5, 5, 5, 5, None, 5], pa.int64())})
    right = pa.table({"k": pa.array([1.0, None, float("nan"), 0.0, 2.0, 2.0], pa.float64()),
                      "t": pa.array([1, 1, 1, 2, 4, None], pa.int64()), "r": ["a", "b", "c", "d", "e", "f"]})
    out = A.asof_join(left, right, ["k"], "t", how="left_outer")
    # a NULL / NaN key never matches; -0.0 meets 0.0; a NULL left t matches nothing; a NULL right t is no candidate
    assert out.column("r").to_pylist() == ["a", None, None, "d", None, "e"]
    assert A.asof_join(left, right, ["k"], "t").column("r").to_pylist() == ["a", "d", "e"]
    fl = pa.table({"t": pa.array([float("nan"), -0.0, 1.5], pa.float64())})
    fr = pa.table({"t": pa.array([0.0, float("nan"), 1.0], pa.float64()), "r": [0, 1, 2]})
    assert A.asof_join(fl, fr, [], "t", how="left_outer").column("r").to_pylist() == [None, 0, 2]
    # strings compare by value
    sl = pa.table({"s": pa.array(["x", "y", "z"]).dictionary_encode(), "t": [3, 3, 3]})
    sr = pa.table({"s": pa.array(["z", "x"]).dictionary_encode(), "t": [1, 2], "r": [0, 1]})
    assert A.asof_join(sl, sr, ["s"], "t", how="left_outer").column("r").to_pylist() == [1, None, 0]


def test_oracle_exact_distances():
    lo, hi = -(1 << 63), (1 << 63) - 1
    tol = hi  # 2^63 - 1: the left row 0 is one unit too far from INT64_MIN, the row -1 is not
    assert A.match_rows([()] * 3, [0, -1, hi], [()], [lo], "backward", True, tol) == [-1, 0, -1]
    got = A.match_rows_np(np.zeros(3, np.int64), np.array([0, -1, hi], np.int64), np.ones(3, bool),
                          np.zeros(1, np.int64), np.array([lo], np.int64), np.ones(1, bool), "backward", True, tol)
    assert got.tolist() == [-1, 0, -1]
    inf = float("inf")
    assert A.match_rows([()], [inf], [()] * 2, [1.0, inf], "nearest", True, 0.5) == [1]


class _DF:
    def __init__(self, expr: str):
        self.schema = Schema(expr)
        self.columns = self.schema.names


def test_schema_rule():
    a, b = _DF("k:long,t:datetime,v:double"), _DF("k:long,t:datetime,q:str,w:int")
    on, s = get_asof_schemas(a, b, ["k"], "t")
    assert on == ["k"] and str(s) == "k:long,t:datetime,v:double,q:str,w:int"
    assert get_asof_schemas(a, b, None, "t")[0] == ["k"]  # None: the common columns but the as-of column
    assert str(get_asof_schemas(a, _DF("t:datetime,q:str"), [], "t")[1]) == "k:long,t:datetime,v:double,q:str"
    with pytest.raises(SchemaError):  # k is common but not a key
        get_asof_schemas(a, b, [], "t")
    with pytest.raises(SchemaError):
        get_asof_schemas(a, _DF("k:int,t:datetime"), ["k"], "t")
    with pytest.raises(SchemaError):
        get_asof_schemas(a, _DF("k:long,t:long"), ["k"], "t")
    with pytest.raises(SchemaError):
        get_asof_schemas(a, _DF("k:long,u:datetime"), ["k"], "t")
    with pytest.raises(ValueError):
        get_asof_schemas(a, b, ["k", "t"], "t")
    with pytest.raises(ValueError):
        get_asof_schemas(a, b, ["k"], ["t"])


def test_key_classes_and_tolerance():
    assert asof_key_class("t", pa.float16(), False) == K.RANGE_KEY_F64
    assert asof_key_class("t", pa.uint64(), False) == K.RANGE_KEY_U64
    for tp in (pa.int8(), pa.date32(), pa.date64(), pa.timestamp("ns", "UTC"), pa.duration("s"), pa.time64("us")):
        assert asof_key_class("t", tp, False) == K.RANGE_KEY_I64
    for tp, is_str in ((pa.string(), True), (pa.bool_(), False), (pa.time32("s"), False)):
        with pytest.raises(ValueError):
            asof_key_class("t", tp, is_str)
    assert asof_tolerance("t", pa.timestamp("us"), datetime.timedelta(seconds=2)) == 2_000_000
    assert asof_tolerance("t", pa.timestamp("ns"), datetime.timedelta(microseconds=3)) == 3000
    assert asof_tolerance("t", pa.date32(), datetime.timedelta(days=2)) == 2
    assert asof_tolerance("t", pa.int64(), 7) == 7 and asof_tolerance("t", pa.float32(), 1) == 1.0
    assert asof_tolerance("t", pa.int64(), None) is None and asof_tolerance("t", pa.int64(), 0) == 0
    for tp, tol in ((pa.int64(), 1.5), (pa.int64(), datetime.timedelta(1)), (pa.int64(), -1), (pa.int64(), True),
                    (pa.timestamp("s"), datetime.timedelta(milliseconds=1)), (pa.float64(), float("inf")),
                    (pa.int64(), 1 << 63)):
        with pytest.raises(ValueError):
            asof_tolerance("t", tp, tol)


class _Engine:
    """Records the as-of calls the SQL engine makes."""
    is_distributed = False

    def __init__(self):
        self.calls = []

    def to_df(self, df):
        return df

    def asof_join(self, df1, df2, **kw):
        self.calls.append((df1, df2, kw))
        return df1

    def join(self, df1, df2, **kw):
        raise AssertionError("an ASOF join must not reach the hash join")


@pytest.mark.parametrize("cond,direction,exact", [
    ("ON a.k = b.k AND a.t >= b.t", "backward", True),
    ("ON a.k = b.k AND a.t > b.t", "backward", False),
    ("ON a.k = b.k AND a.t <= b.t", "forward", True),
    ("ON a.t < b.t AND a.k = b.k", "forward", False),
    ("ON b.t <= a.t AND a.k = b.k", "backward", True),
    ("ON b.t < a.t AND b.k = a.k", "backward", False),
    ("ON (a.k = b.k) AND (b.t >= a.t)", "forward", True),
    ("USING (k, t)", "backward", True),
])
def test_sql_forms(cond, direction, exact):
    from fugue_b200.sql import B200SQLEngine

    eng = _Engine()
    ta, tb = _DF("k:long,t:long,v:double"), _DF("k:long,t:long,w:double")
    for kind, how in (("", "inner"), ("LEFT ", "left_outer"), ("LEFT OUTER ", "left_outer"), ("INNER ", "inner")):
        B200SQLEngine(eng).select({"ta": ta, "tb": tb}, f"SELECT * FROM ta AS a ASOF {kind}JOIN tb b {cond}")
        d1, d2, kw = eng.calls[-1]
        assert d1 is ta and d2 is tb
        assert kw == dict(on=["k"], asof="t", how=how, direction=direction, allow_exact_matches=exact)
    B200SQLEngine(eng).select({"ta": ta, "tb": tb}, "SELECT * FROM ta ASOF JOIN tb ON ta.t >= tb.t")
    assert eng.calls[-1][2]["on"] == [] and eng.calls[-1][2]["direction"] == "backward"
    # qualifiers that name no table (dataframes handed to raw_sql get generated names) are in FROM order, or take
    # the side the other operand leaves
    for c, d in (("trades.t >= quotes.t", "backward"), ("trades.t < quotes.t", "forward"), ("b.t < x.t", "backward"),
                 ("x.t <= a.t", "backward")):
        B200SQLEngine(eng).select({"ta": ta, "tb": tb}, f"SELECT * FROM ta a ASOF JOIN tb b ON x.k = y.k AND {c}")
        assert eng.calls[-1][2]["direction"] == d, c


@pytest.mark.parametrize("sql", [
    "SELECT a.v FROM ta a ASOF JOIN tb b ON a.k = b.k AND a.t >= b.t",
    "SELECT * FROM ta a ASOF RIGHT JOIN tb b ON a.k = b.k AND a.t >= b.t",
    "SELECT * FROM ta a ASOF FULL OUTER JOIN tb b ON a.k = b.k AND a.t >= b.t",
    "SELECT * FROM ta a ASOF JOIN tb b ON a.t >= b.t AND a.t <= b.t",
    "SELECT * FROM ta a ASOF JOIN tb b ON a.k = b.k",
    "SELECT * FROM ta a ASOF JOIN tb b ON a.k = b.k AND t >= t",
    "SELECT * FROM ta a ASOF JOIN tb b ON a.t >= a.t",
    "SELECT * FROM ta a ASOF JOIN tb b ON a.k = b.j AND a.t >= b.t",
    "SELECT * FROM ta a ASOF JOIN tb b",
    "SELECT * FROM ta a ASOF JOIN tb b ON a.k = a.k AND a.t >= b.t",         # an equality within one table
])
def test_sql_rejections(sql):
    from fugue_b200.sql import B200SQLEngine

    eng = _Engine()
    with pytest.raises(NotImplementedError):
        B200SQLEngine(eng).select({"ta": _DF("k:long,t:long"), "tb": _DF("k:long,t:long,j:long")}, sql)
    assert eng.calls == []


def test_engine_rejections_before_the_device():
    import torch

    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.dist import DistributedB200Engine
    from fugue_b200.execution_engine import B200ExecutionEngine
    from fugue_b200.table import B200Table

    def table(s):  # host tensors: nothing may reach the device
        return B200DataFrame(B200Table(Schema("k:long,s:str"), [torch.tensor([1]), torch.tensor([0], dtype=torch.int32)],
                                       [None, None], {"s": pa.array([s])}))

    a, b = table("x"), table("y")
    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)
    eng.to_df = lambda df, schema=None: df  # type: ignore
    eng.get_current_parallelism = lambda: 1  # type: ignore
    with pytest.raises(ValueError, match="numeric or temporal"):  # a string as-of column
        eng.asof_join(a, b, on=["k"], asof="s")
    for kw in (dict(how="right_outer"), dict(how="cross"), dict(direction="sideways"),
               dict(allow_exact_matches=None)):
        with pytest.raises(ValueError):
            eng.asof_join(a, b, on=["k"], asof="s", **kw)
    dist = DistributedB200Engine.__new__(DistributedB200Engine)
    dist._world = 2
    dist.to_df = lambda df, schema=None: (_ for _ in ()).throw(AssertionError("must reject first"))  # type: ignore
    with pytest.raises(NotImplementedError, match="multi-GPU"):
        dist.asof_join(None, None, on=["k"], asof="t")
