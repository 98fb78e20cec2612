"""Window functions of a ColumnMap (K9) on the H100: the segmented-scan kernel ``fb_segmented_scan`` against
oracle/window.py (every op, tile and carry-chunk boundaries, segment shapes, NULLs, wrap-around, totalOrder,
bit-exact and bounded float sums, determinism), then whole maps through ``fa.transform`` against the oracle and
against ``engine.aggregate``."""
import math
from collections import OrderedDict

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import all_cols, col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.execution_engine import B200ExecutionEngine
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import window as W

DEV = torch.device("cuda", 0)
OPS = {"SUM_I64": K.AGG_SUM_I64, "SUM_F64": K.AGG_SUM_F64, "MIN_I64": K.AGG_MIN_I64, "MAX_I64": K.AGG_MAX_I64,
       "MIN_F64": K.AGG_MIN_F64, "MAX_F64": K.AGG_MAX_F64, "COUNT": K.AGG_COUNT}
TILE = 2048  # rows per CTA of fb_segscan_tile_kernel<OpScan, ...>; 1024 * TILE rows fill one pass of the carry kernel


def _offsets(n: int, shape: str, rng) -> np.ndarray:
    if n == 0:
        return np.array([0, 0], dtype=np.int64)
    if shape == "singletons":
        return np.arange(n + 1, dtype=np.int64)
    if shape == "spanning":
        return np.array([0, n], dtype=np.int64)
    if shape == "zipf":  # lengths Zipf-skewed, plus empty segments
        lens = np.minimum(rng.zipf(1.3, n), n)
        lens[rng.random(n) < 0.05] = 0
        cut = np.concatenate([[0], np.cumsum(lens)])
        cut = cut[cut < n]
        return np.concatenate([cut, [n, n]]).astype(np.int64)
    raise ValueError(shape)


def _values(op: str, n: int, rng) -> np.ndarray:
    if op == "SUM_F64":  # finite: inf - inf orders differ between any two summation orders
        return rng.standard_normal(n).view(np.int64)
    if op.endswith("F64"):
        special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -1.5], dtype=np.float64)
        x = np.where(rng.random(n) < 0.2, rng.choice(special, n), rng.standard_normal(n))
        bits = x.view(np.int64).copy()
        neg_nan = rng.random(n) < 0.02  # NaN with the sign bit set and a payload
        bits[neg_nan] = np.int64(-0x0007FFFF00000001)
        return bits
    return rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64, endpoint=True)


def _run(offsets, cols):
    d_off = torch.from_numpy(offsets).to(DEV)
    n = int(offsets[-1])
    spec = [(OPS[op], None if v is None or op == "COUNT" else torch.from_numpy(v).to(DEV),
             None if m is None else torch.from_numpy(m.astype(np.uint8)).to(DEV)) for op, v, m in cols]
    res = K.segmented_scan(d_off, n, spec)
    torch.cuda.synchronize()
    return [(None if o is None else o.view(torch.int64).cpu().numpy(), c.cpu().numpy()) for o, c in res]


@pytest.mark.parametrize("n", [0, 1, 7, TILE - 1, TILE, TILE + 1, 5 * TILE + 3, 1024 * TILE + 1, 3_000_017])
@pytest.mark.parametrize("shape", ["singletons", "zipf", "spanning"])
def test_kernel_matches_oracle_for_every_op(n, shape):
    rng = np.random.default_rng(n * 7 + len(shape))
    offsets = _offsets(n, shape, rng)
    cols = []
    for op in OPS:
        v = _values(op, n, rng)
        for with_valid in (False, True):
            m = None
            if with_valid:
                m = rng.random(n) < 0.7
                if len(offsets) > 2:  # an all-NULL segment
                    m[offsets[1]:offsets[2]] = False
            cols.append((op, v, m))
    got = _run(offsets, cols)  # 14 scans: two launch sequences of up to 8 columns
    for (op, v, m), (gv, gc) in zip(cols, got):
        ev, ec = W.segmented_scan(v, m, offsets, op)
        assert np.array_equal(gc, ec), (op, m is not None)
        if op == "SUM_F64":
            ok = ec > 0
            a, b = gv.view(np.float64)[ok], ev.view(np.float64)[ok]
            fin = np.isfinite(b)
            assert np.allclose(a[fin], b[fin], rtol=1e-6, atol=1e-6) and np.array_equal(np.isnan(a), np.isnan(b))
        elif op != "COUNT":
            assert np.array_equal(gv, ev), (op, m is not None)


def test_f64_sum_is_exact_where_every_prefix_is_and_bounded_otherwise():
    rng = np.random.default_rng(5)
    n = 3_000_000
    exact = (rng.integers(-(2**30), 2**30, n) * 2.0 ** -10)  # multiples of 2^-10 below 2^20
    for shape in ("spanning", "zipf"):
        off = _offsets(n, shape, rng)
        (gv, _), = _run(off, [("SUM_F64", exact.view(np.int64), None)])
        ev, _ = W.segmented_scan(exact.view(np.int64), None, off, "SUM_F64")
        assert np.array_equal(gv, ev), shape
    x = rng.standard_normal(n)
    off = np.array([0, 17, 5000, 5001, 1_000_000, n], dtype=np.int64)
    (gv, _), = _run(off, [("SUM_F64", x.view(np.int64), None)])
    g = gv.view(np.float64)
    for s, e in zip(off[:-1], off[1:]):
        m = e - s
        seg = x[s:e]
        bound = (m - 1) * 2.0 ** -52 * float(np.abs(seg).sum())
        assert abs(g[e - 1] - math.fsum(seg)) <= bound, (s, e)


def test_runs_are_bit_identical():
    rng = np.random.default_rng(11)
    n = 3_000_000
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
    off = np.array([0, n], dtype=np.int64)
    first = _run(off, [("SUM_F64", x.view(np.int64), None)])[0][0]
    second = _run(off, [("SUM_F64", x.view(np.int64), None)])[0][0]
    assert np.array_equal(first, second)


def test_int64_sum_wraps_around():
    n = 3 * TILE + 5
    v = np.full(n, 2**62 + 12345, dtype=np.int64)
    off = np.array([0, 10, n], dtype=np.int64)
    (gv, _), = _run(off, [("SUM_I64", v, None)])
    ev, _ = W.segmented_scan(v, None, off, "SUM_I64")
    assert np.array_equal(gv, ev) and (ev < 0).any()


# ---- through fa.transform ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _input(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    m = lambda q: rng.random(n) < q  # noqa: E731
    keyf = np.array([1.5, 2.25, -3.0, 7.0, 100.5])[rng.integers(0, 5, n)]
    return pa.table({
        "rid": pa.array(np.arange(n)),
        "k": pa.array(rng.integers(0, 40, n), mask=m(0.05)),
        "k2": pa.array(rng.integers(0, 3, n).astype(np.int32), mask=m(0.1)),
        "kf": pa.array(keyf, mask=m(0.05)),
        "ks": pa.array(list(np.array(["x", "y", "z", "w"], dtype=object)[rng.integers(0, 4, n)]), mask=m(0.05),
                       type=pa.string()),
        "kd": pa.array(rng.integers(18000, 18010, n).astype(np.int32), mask=m(0.05)).cast(pa.date32()),
        "p": pa.array(rng.integers(0, 8, n), mask=m(0.1)),
        "q": pa.array(np.round(rng.standard_normal(n), 1) + 0.05, mask=m(0.1)),
        "v": pa.array(rng.integers(-1000, 1000, n), mask=m(0.2)),
        "i": pa.array(rng.integers(-(2**62), 2**62, n), mask=m(0.1)),
        "x": pa.array(rng.standard_normal(n), mask=m(0.2)),
        "s": pa.array(list(np.array(["a", "b", "c"], dtype=object)[rng.integers(0, 3, n)]), mask=m(0.2),
                      type=pa.string()),
    })


ALL = [f.row_number().alias("rn"), f.rank().alias("rk"), f.dense_rank().alias("dr"),
       f.sum(col("v")).over(running=True).alias("rsv"), f.sum(col("v")).over().alias("tsv"),
       f.sum(col("i")).over(running=True).alias("rsi"), f.sum(col("x")).over(running=True).alias("rsx"),
       f.sum(col("x")).over().alias("tsx"), f.avg(col("v")).over(running=True).alias("rav"),
       f.avg(col("x")).over().alias("tav"), f.count(col("v")).over(running=True).alias("rcv"),
       f.count(all_cols()).over().alias("cnt"), f.min(col("x")).over(running=True).alias("rmin"),
       f.max(col("x")).over().alias("tmax"), f.min(col("v")).over().alias("tminv"),
       f.max(col("i")).over(running=True).alias("rmaxi"), f.first(col("s")).over(running=True).alias("rfs"),
       f.first(col("x")).over().alias("tfx"), f.last(col("v")).over(running=True).alias("ffill"),
       f.last(col("s")).over().alias("tls"), f.lag(col("v")).alias("lag"), f.lead(col("x"), 2).alias("lead2"),
       f.lag(col("s"), 1, "none").alias("lags"), f.lead(col("v"), 0).alias("same"),
       f.lag(col("v"), 3, -7).alias("lag3")]
ALL_SCHEMA = ("rid:long,rn:long,rk:long,dr:long,rsv:long,tsv:long,rsi:long,rsx:double,tsx:double,rav:double,"
              "tav:double,rcv:long,cnt:long,rmin:double,tmax:double,tminv:long,rmaxi:long,rfs:str,tfx:double,"
              "ffill:long,tls:str,lag:long,lead2:double,lags:str,same:long,lag3:long")
APPROX = {"rsx", "tsx", "rav", "tav", "share"}  # float sums: the kernel does not add in row order


def _check(engine, t: pa.Table, keys, presort: OrderedDict, cols, schema: str, **spec):
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    ps = ",".join(f"{k} {'asc' if a else 'desc'}" for k, a in presort.items())
    res = fa.transform(df, ColumnMap(col("rid"), *cols), schema=schema,
                       partition=PartitionSpec(by=keys, presort=ps, **spec), engine=engine, as_fugue=True)
    got = res.as_arrow()
    assert got.num_rows == t.num_rows
    order = np.argsort(np.asarray(got.column("rid")))
    exp = W.window_map(t, keys, presort, [col("rid")] + list(cols))
    for name in got.column_names:
        g = [got.column(name)[int(i)].as_py() for i in order]
        e = exp[name]
        if name in APPROX:
            assert [x is None for x in g] == [x is None for x in e], name
            assert np.allclose([x for x in g if x is not None], [x for x in e if x is not None], rtol=1e-9,
                               atol=1e-9), name
        else:
            assert g == e, name
    return res


@pytest.mark.parametrize("algo,num", [("hash", 16), ("even", 4), ("rand", 3), ("hash", 0)])
def test_every_window_function_against_the_oracle(engine, algo, num):
    t = _input(3000, 1)
    _check(engine, t, ["k"], OrderedDict(p=True, q=False), ALL, ALL_SCHEMA, algo=algo, num=num)


@pytest.mark.parametrize("keys", [["kf"], ["ks"], ["kd"], ["k2", "ks"], []])
def test_key_types_and_no_keys(engine, keys):
    t = _input(2000, 2)
    _check(engine, t, keys, OrderedDict(p=False), ALL, ALL_SCHEMA)


@pytest.mark.parametrize("presort", [OrderedDict(), OrderedDict(q=True), OrderedDict(q=False),
                                     OrderedDict(p=False, s=True)])
def test_presort_directions_nulls_and_ties(engine, presort):
    t = _input(2500, 3)
    _check(engine, t, ["k"], presort, ALL, ALL_SCHEMA)


def test_window_nodes_inside_expressions(engine):
    t = _input(2000, 4)
    cols = [(col("x") / f.sum(col("x")).over()).alias("share"), (col("v") - f.lag(col("v"))).alias("dv"),
            (f.row_number() * 10 + f.dense_rank()).alias("code"),
            f.sum(col("v") * 2 + 1).over(running=True).alias("rs2"), f.max(col("p")).over().cast(float).alias("mp")]
    res = _check(engine, t, ["k"], OrderedDict(p=True), cols, "rid:long,share:double,dv:long,code:long,rs2:long,mp:double")
    assert res.native.partition_keys is None  # the key is not an output column


def test_partition_values_equal_aggregate(engine):
    t = _input(20000, 5)
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    cols = [f.min(col("x")).over().alias("mn"), f.max(col("i")).over().alias("mx"), f.sum(col("i")).over().alias("si"),
            f.sum(col("x")).over().alias("sx"), f.count(col("v")).over().alias("c"), f.max(col("x")).over().alias("mxx")]
    res = fa.transform(df, ColumnMap("k", *cols), schema="k:long,mn:double,mx:long,si:long,sx:double,c:long,mxx:double",
                       partition=PartitionSpec(by="k"), engine=engine, as_fugue=True)
    assert res.native.partition_keys == ["k"]
    win = res.as_pandas().drop_duplicates("k").set_index("k").sort_index()
    agg = engine.aggregate(df, PartitionSpec(by="k"), [f.min(col("x")).alias("mn"), f.max(col("i")).alias("mx"),
                                                       f.sum(col("i")).alias("si"), f.sum(col("x")).alias("sx"),
                                                       f.count(col("v")).alias("c"), f.max(col("x")).alias("mxx")])
    agg = agg.as_pandas().set_index("k").sort_index()
    assert len(win) == len(agg)
    for c in ["mn", "mxx"]:
        assert np.array_equal(win[c].to_numpy().view(np.int64), agg[c].to_numpy().view(np.int64)), c
    for c in ["mx", "si", "c"]:
        assert np.array_equal(win[c].to_numpy(), agg[c].to_numpy()), c
    assert np.allclose(win["sx"], agg["sx"], rtol=1e-12, atol=1e-12)


def test_unsupported_layouts_raise(engine):
    t = _input(100, 6)
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    cm = ColumnMap("rid", f.row_number().alias("rn"))
    with pytest.raises(NotImplementedError):
        fa.transform(df, cm, schema="rid:long,rn:long", partition=PartitionSpec(by="k", algo="coarse"), engine=engine)
    with pytest.raises(NotImplementedError):
        fa.transform(df, cm, schema="rid:long,rn:long", partition=PartitionSpec(num=4), engine=engine)
    with pytest.raises(NotImplementedError):
        fa.transform(df, ColumnMap("rid", f.sum(col("s")).over().alias("x")), schema="rid:long,x:long",
                     partition=PartitionSpec(by="k"), engine=engine)

    class _MultiGpu(B200ExecutionEngine):
        @property
        def is_distributed(self) -> bool:
            return True

    with pytest.raises(NotImplementedError):
        fa.transform(df, cm, schema="rid:long,rn:long", partition=PartitionSpec(by="k"), engine=_MultiGpu())
