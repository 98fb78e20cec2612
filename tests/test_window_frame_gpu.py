"""Moving frames (ROWS BETWEEN) on the H100: the kernel ``fb_window_frame`` against tests/_frame_oracle.py (every
op, NULLs, segment shapes, sizes around the CTA tiles, frames on both sides of ``FRAME_TILE_MAX_WIDTH``,
exact integer / MIN / MAX results, f64 sums bit-exact where every partial sum is exact and within the frame's
error bound otherwise, cancellation, repeat runs, extreme bounds), then whole maps through ``fa.transform``."""
import math
from collections import OrderedDict

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import _lib
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import all_cols, col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table

import _frame_oracle as F  # noqa: E402

DEV = torch.device("cuda", 0)
OPS = {"SUM_I64": K.AGG_SUM_I64, "SUM_F64": K.AGG_SUM_F64, "MIN_I64": K.AGG_MIN_I64, "MAX_I64": K.AGG_MAX_I64,
       "MIN_F64": K.AGG_MIN_F64, "MAX_F64": K.AGG_MAX_F64, "COUNT": K.AGG_COUNT}
TW = K.FRAME_TILE_MAX_WIDTH
SPAN = 2 * TW  # rows staged per CTA of the one-pass kernel; 2048 is also the scan's tile
FRAMES = [(-2, 0), (-1, 1), (0, 0), (1, 3), (-5, -1), (None, -1), (None, 2), (0, None), (-3, None),
          (-(TW - 1), 0), (-TW, 0), (-(TW // 2), TW // 2), (3, TW + 3)]
I64_MIN, I64_MAX = -(2**63), 2**63 - 1


def _offsets(n: int, shape: str, rng) -> np.ndarray:
    if n == 0:
        return np.array([0, 0], dtype=np.int64)
    if shape == "singletons":
        return np.arange(n + 1, dtype=np.int64)
    if shape == "spanning":
        return np.array([0, n], dtype=np.int64)
    if shape == "short":  # 1 to 4 rows: (5, 7) is empty on every row
        cut = np.concatenate([[0], np.cumsum(rng.integers(1, 5, n))])
        return np.concatenate([cut[cut < n], [n]]).astype(np.int64)
    if shape == "zipf":  # lengths Zipf-skewed, plus empty segments
        lens = np.minimum(rng.zipf(1.3, n), n)
        lens[rng.random(n) < 0.05] = 0
        cut = np.concatenate([[0], np.cumsum(lens)])
        cut = cut[cut < n]
        return np.concatenate([cut, [n, n]]).astype(np.int64)
    raise ValueError(shape)


def _values(op: str, n: int, rng) -> np.ndarray:
    if op == "SUM_F64":  # multiples of 2^-10 below 2^20: every partial sum is exact, so any order is bit-exact
        return (rng.integers(-(2**30), 2**30, n) * 2.0 ** -10).view(np.int64)
    if op.endswith("F64"):
        special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -1.5], dtype=np.float64)
        x = np.where(rng.random(n) < 0.2, rng.choice(special, n), rng.standard_normal(n))
        bits = x.view(np.int64).copy()
        bits[rng.random(n) < 0.02] = np.int64(-0x0007FFFF00000001)  # NaN with the sign bit set and a payload
        return bits
    return rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)


def _columns(n: int, offsets: np.ndarray, rng):
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
    return cols


def _run(offsets, start, end, cols):
    d_off = torch.from_numpy(offsets).to(DEV)
    n = int(offsets[-1])
    spec = [(OPS[op], None if op == "COUNT" else torch.from_numpy(v).to(DEV),
             None if m is None else torch.from_numpy(m.astype(np.uint8)).to(DEV)) for op, v, m in cols]
    res = K.window_frame(d_off, n, start, end, spec)
    torch.cuda.synchronize()
    return [(None if o is None else o.view(torch.int64).cpu().numpy(), c.cpu().numpy()) for o, c in res]


def _check(offsets, frame, cols, got):
    for (op, v, m), (gv, gc) in zip(cols, got):
        ev, ec = F.frame_aggregate(None if op == "COUNT" else v, m, offsets, op, *frame, loop=False)
        assert np.array_equal(gc, ec), (op, frame, m is not None)
        if op != "COUNT":  # integers, MIN / MAX and exact f64 sums: bit for bit
            assert np.array_equal(gv, ev), (op, frame, m is not None)


@pytest.mark.parametrize("n", [0, 1, SPAN - 1, SPAN, SPAN + 1, 5 * SPAN + 3])
@pytest.mark.parametrize("shape", ["singletons", "zipf", "spanning"])
def test_kernel_matches_oracle_for_every_op_and_frame(n, shape):
    rng = np.random.default_rng(n * 7 + len(shape))
    offsets = _offsets(n, shape, rng)
    cols = _columns(n, offsets, rng)
    for frame in FRAMES:
        _check(offsets, frame, cols, _run(offsets, *frame, cols))  # 14 columns: two launch sequences


@pytest.mark.parametrize("shape", ["zipf", "spanning"])
def test_three_million_rows(shape):
    rng = np.random.default_rng(17 + len(shape))
    n = 3_000_017
    offsets = _offsets(n, shape, rng)
    cols = _columns(n, offsets, rng)
    for frame in [(-2, 0), (-1, 1), (1, 3), (None, -1), (0, None), (-3, None)]:
        _check(offsets, frame, cols, _run(offsets, *frame, cols))


def test_both_sides_of_the_tile_limit_at_scale():
    rng = np.random.default_rng(23)
    n = 60_003
    offsets = _offsets(n, "zipf", rng)
    cols = _columns(n, offsets, rng)
    for frame in [(-(TW - 1), 0), (-TW, 0), (-(TW // 2) + 1, TW // 2), (-(TW // 2), TW // 2 + 1)]:
        _check(offsets, frame, cols, _run(offsets, *frame, cols))


def test_frames_wider_than_every_segment_and_empty_for_whole_segments():
    rng = np.random.default_rng(29)
    n = 8_000
    offsets = _offsets(n, "short", rng)
    cols = _columns(n, offsets, rng)
    for frame in [(-10, 10), (-TW, TW), (5, 7), (-9, -5), (4, None), (None, -4), (-100, -5)]:
        got = _run(offsets, *frame, cols)
        _check(offsets, frame, cols, got)
        if frame in [(5, 7), (-9, -5), (4, None), (None, -4), (-100, -5)]:
            assert all((c == 0).all() for _, c in got), frame


def test_f64_sum_is_within_the_frame_bound():
    rng = np.random.default_rng(31)
    n = 1_000_003
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)
    offsets = _offsets(n, "zipf", rng)
    ok = rng.random(n) < 0.9
    sample = np.sort(rng.choice(n, 1500, replace=False))
    for frame in [(-6, 0), (-2, 2), (-TW, 0), (None, 2), (-3, None)]:
        (gv, gc), = _run(offsets, *frame, [("SUM_F64", x.view(np.int64), ok)])
        g = gv.view(np.float64)
        lo, hi = F.frame_bounds(offsets, *frame)
        for i in sample.tolist():
            vals = x[lo[i]:hi[i] + 1][ok[lo[i]:hi[i] + 1]] if hi[i] >= lo[i] else x[:0]
            assert gc[i] == len(vals)
            bound = max(len(vals) - 1, 0) * 2.0 ** -52 * float(np.abs(vals).sum())
            assert abs(g[i] - math.fsum(vals.tolist())) <= bound, (frame, i)


def test_a_large_value_does_not_spoil_later_frames():
    n = 3 * SPAN + 11
    x = np.ones(n)
    x[0] = 1e20
    offsets = np.array([0, n], dtype=np.int64)
    (gv, gc), = _run(offsets, -2, 0, [("SUM_F64", x.view(np.int64), None)])
    assert (gv.view(np.float64)[3:] == 3.0).all() and (gc[2:] == 3).all()
    (gv, _), = _run(offsets, -TW, 0, [("SUM_F64", x.view(np.int64), None)])  # wider than the tile: the scan path
    assert (gv.view(np.float64)[TW + 1:] == TW + 1.0).all()


def test_runs_are_bit_identical():
    rng = np.random.default_rng(37)
    n = 3_000_000
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
    offsets = _offsets(n, "zipf", rng)
    for frame in [(-6, 0), (-TW, 0), (None, 5)]:
        first = _run(offsets, *frame, [("SUM_F64", x.view(np.int64), None)])[0][0]
        second = _run(offsets, *frame, [("SUM_F64", x.view(np.int64), None)])[0][0]
        assert np.array_equal(first, second), frame


def _raw(offsets, start, end, flags, v):
    """fb_window_frame called directly: the bounds reach the C ABI unchanged."""
    lib = _lib.load()
    n = int(offsets[-1])
    d_off = torch.from_numpy(offsets).to(DEV)
    dv = torch.from_numpy(v).to(DEV)
    out = torch.empty_like(dv)
    cnt = torch.empty(n, dtype=torch.int64, device=DEV)
    nb = int(lib.fb_window_frame_scratch_bytes(n, 1, start, end, flags))
    scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=DEV)
    _lib.check(lib.fb_window_frame(DEV.index, torch.cuda.current_stream(DEV).cuda_stream, n, len(offsets) - 1,
                                   d_off.data_ptr(), start, end, flags, 1, _lib.i32_array([K.AGG_SUM_I64]),
                                   _lib.ptr_array([dv.data_ptr()]), _lib.ptr_array([0]),
                                   _lib.ptr_array([out.data_ptr()]), _lib.ptr_array([cnt.data_ptr()]),
                                   scratch.data_ptr(), scratch.numel()))
    torch.cuda.synchronize()
    return out.cpu().numpy(), cnt.cpu().numpy()


def test_extreme_bounds_and_rejection():
    rng = np.random.default_rng(41)
    n = 10_000
    offsets = _offsets(n, "zipf", rng)
    v = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    cases = {(I64_MIN + 1, I64_MAX): (None, None), (I64_MIN + 1, -1): (None, -1), (1, I64_MAX): (1, None),
             (I64_MIN + 1, I64_MIN + 1): (I64_MIN + 1, I64_MIN + 1), (I64_MAX, I64_MAX): (I64_MAX, I64_MAX),
             (I64_MIN, I64_MAX): (None, None), (-n, n): (None, None), (-(n - 1), n - 1): (-(n - 1), n - 1)}
    for (s, e), frame in cases.items():
        got = _raw(offsets, s, e, 0, v)
        ev, ec = F.frame_aggregate(v, None, offsets, "SUM_I64", *frame, loop=False)
        assert np.array_equal(got[1], ec) and np.array_equal(got[0], ev), (s, e)
    # an unbounded side ignores its bound
    got = _raw(offsets, I64_MAX, -3, K.FRAME_UNBOUNDED_START, v)
    ev, ec = F.frame_aggregate(v, None, offsets, "SUM_I64", None, -3, loop=False)
    assert np.array_equal(got[0], ev) and np.array_equal(got[1], ec)
    with pytest.raises(_lib.FugueB200KernelError):
        _raw(offsets, 1, 0, 0, v)
    with pytest.raises(_lib.FugueB200KernelError):
        _raw(offsets, I64_MAX, I64_MIN, 0, v)


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


FR = [f.sum(col("v")).over(rows=(-2, 0)).alias("s3"), f.sum(col("x")).over(rows=(-6, 0)).alias("sx7"),
      f.avg(col("v")).over(rows=(-2, 2)).alias("av5"), f.count(col("v")).over(rows=(1, 5)).alias("cn"),
      f.count(all_cols()).over(rows=(-3, -1)).alias("cs"), f.min(col("x")).over(rows=(-1, 1)).alias("mn"),
      f.max(col("i")).over(rows=(0, None)).alias("mxi"), f.max(col("x")).over(rows=(None, -1)).alias("mxp"),
      f.first(col("s")).over(rows=(-2, 0)).alias("fs"), f.last(col("v")).over(rows=(0, 3)).alias("lv"),
      f.last(col("s")).over(rows=(None, 1)).alias("ls"), f.sum(col("i")).over(rows=(-TW, 0)).alias("wide"),
      f.min(col("v")).over(rows=(-3, None)).alias("mnv"), f.sum(col("v")).over(rows=(5, 7)).alias("ahead"),
      (col("v") - f.avg(col("v")).over(rows=(-6, 0))).alias("dev")]
FR_SCHEMA = ("rid:long,s3:long,sx7:double,av5:double,cn:long,cs:long,mn:double,mxi:long,mxp:double,fs:str,lv:long,"
             "ls:str,wide:long,mnv:long,ahead:long,dev:double")
APPROX = {"sx7", "av5", "dev"}  # float sums: the kernel does not add in row order


def _check_map(engine, t: pa.Table, keys, presort: OrderedDict, cols, schema: str, **spec):
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    ps = ",".join(f"{k} {'asc' if a else 'desc'}" for k, a in presort.items())
    res = fa.transform(df, ColumnMap(col("rid"), *cols), schema=schema,
                       partition=PartitionSpec(by=keys, presort=ps, **spec), engine=engine, as_fugue=True)
    got = res.as_arrow()
    assert got.num_rows == t.num_rows
    order = np.argsort(np.asarray(got.column("rid")))
    exp = F.window_map(t, keys, presort, [col("rid")] + list(cols))
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


@pytest.mark.parametrize("algo,num", [("hash", 16), ("even", 4), ("rand", 3)])
def test_every_frame_column_against_the_oracle(engine, algo, num):
    t = _input(3000, 1)
    res = _check_map(engine, t, ["k"], OrderedDict(p=True, q=False), FR, FR_SCHEMA, algo=algo, num=num)
    assert "fs" in res.native.dictionaries and "ls" in res.native.dictionaries  # strings keep their dictionary


@pytest.mark.parametrize("keys", [["kf"], ["ks"], ["kd"], ["k2", "ks"], []])
def test_key_types_and_no_keys(engine, keys):
    _check_map(engine, _input(2000, 2), keys, OrderedDict(p=False), FR, FR_SCHEMA)


@pytest.mark.parametrize("presort", [OrderedDict(), OrderedDict(q=True), OrderedDict(q=False),
                                     OrderedDict(p=False, s=True)])
def test_presort_directions_nulls_and_ties(engine, presort):
    _check_map(engine, _input(2500, 3), ["k"], presort, FR, FR_SCHEMA)


def test_unbounded_frames_equal_running_and_whole(engine):
    t = _input(4000, 4)
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    cols = [f.sum(col("x")).over(rows=(None, 0)).alias("a"), f.sum(col("x")).over(running=True).alias("b"),
            f.max(col("v")).over(rows=(None, None)).alias("c"), f.max(col("v")).over().alias("d"),
            f.first(col("s")).over(rows=(None, None)).alias("e"), f.first(col("s")).over().alias("g")]
    got = fa.transform(df, ColumnMap(col("rid"), *cols), schema="rid:long,a:double,b:double,c:long,d:long,e:str,g:str",
                       partition=PartitionSpec(by="k", presort="p"), engine=engine, as_fugue=True).as_arrow()
    for a, b in (("a", "b"), ("c", "d"), ("e", "g")):
        assert got.column(a).equals(got.column(b)), (a, b)


def test_sum_of_a_string_column_raises(engine):
    df = B200DataFrame(B200Table.from_arrow(_input(100, 6), DEV))
    with pytest.raises(NotImplementedError):
        fa.transform(df, ColumnMap("rid", f.sum(col("s")).over(rows=(-2, 0)).alias("x")), schema="rid:long,x:long",
                     partition=PartitionSpec(by="k"), engine=engine)
