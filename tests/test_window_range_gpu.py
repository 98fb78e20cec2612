"""Value frames (RANGE BETWEEN) on the H100: ``fb_window_range_bounds`` against ``_range_oracle.range_bounds`` (every
key class and direction, ties, NULL tails, segment shapes, 0 to 3 M rows, extreme offsets and keys, uint64 keys
>= 2^63, float keys with +-inf and subnormals), ``fb_window_bounded`` against ``_range_oracle.bounded_aggregate``
(every op, NULLs, arbitrary bounds, one 3 M-row frame set that uses the tree's top levels, exact and
error-bounded f64 sums, repeat runs), then whole maps through ``fa.transform``."""
import datetime
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
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema, type_to_expr
from fugue_b200.table import B200Table

import _range_oracle as R  # noqa: E402

DEV = torch.device("cuda", 0)
OPS = {"SUM_I64": K.AGG_SUM_I64, "SUM_F64": K.AGG_SUM_F64, "MIN_I64": K.AGG_MIN_I64, "MAX_I64": K.AGG_MAX_I64,
       "MIN_F64": K.AGG_MIN_F64, "MAX_F64": K.AGG_MAX_F64, "COUNT": K.AGG_COUNT}
CLS = {"I64": K.RANGE_KEY_I64, "U64": K.RANGE_KEY_U64, "F64": K.RANGE_KEY_F64}
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
TILE = 256  # rows per CTA of the bounds kernel
TD = datetime.timedelta
_ENGINE = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _offsets(n, shape, rng):
    if n == 0:
        return np.array([0, 0], dtype=np.int64)
    if shape == "singletons":
        return np.arange(n + 1, dtype=np.int64)
    if shape == "spanning":
        return np.array([0, n], dtype=np.int64)
    lens = np.minimum(rng.zipf(1.3, n), n)  # zipf, with empty segments
    lens[rng.random(n) < 0.05] = 0
    cut = np.concatenate([[0], np.cumsum(lens)])
    return np.concatenate([cut[cut < n], [n, n]]).astype(np.int64)


def _keys(n, cls, rng, spread):
    if cls == "F64":
        special = np.array([np.inf, -np.inf, 5e-324, -5e-324, 0.0, -0.0, 1e308, -1e308])
        x = np.where(rng.random(n) < 0.1, rng.choice(special, n), np.round(rng.standard_normal(n) * spread) / 4)
        x[rng.random(n) < 0.03] = np.nan  # NULL as a float key
        return x
    if cls == "U64":
        x = rng.integers(0, max(spread, 1), n).astype(np.uint64)
        x[rng.random(n) < 0.3] += np.uint64(2**63)
        x[rng.random(n) < 0.02] = np.uint64(2**64 - 1)
        return x.view(np.int64)
    x = rng.integers(-spread, spread + 1, n).astype(np.int64)
    x[rng.random(n) < 0.02] = I64_MIN
    x[rng.random(n) < 0.02] = I64_MAX
    return x


def _sorted(off, keys, valid, cls, ascending):
    """Sort every segment by key (NULL and NaN last), as the presort leaves it."""
    k, ok = keys.copy(), valid.copy()
    if cls == "F64":
        ok &= ~np.isnan(k)
        order_key = np.where(k == 0, 0.0, k)
    else:
        order_key = k.view(np.uint64) if cls == "U64" else k
    seg = np.repeat(np.arange(len(off) - 1), np.diff(off))
    ranks = np.unique(order_key[ok], return_inverse=True)[1] if ok.any() else np.zeros(0, np.int64)
    r = np.zeros(len(k), dtype=np.int64)
    r[ok] = ranks if ascending else -ranks
    o = np.lexsort((np.arange(len(k)), r, ~ok, seg))
    return k[o], ok[o]


def _bounds(off, k, ok, cls, asc, start, end):
    """The kernel's bounds; with every key valid (float keys: no NaN) the validity goes as NULL."""
    mask = None if ok.all() and not (cls == "F64" and np.isnan(k).any()) else \
        torch.from_numpy(ok.astype(np.uint8)).to(DEV)
    lo, hi = K.window_range_bounds(torch.from_numpy(off).to(DEV), torch.from_numpy(k).to(DEV), mask, CLS[cls], asc,
                                   start, end)
    return lo.cpu().numpy(), hi.cpu().numpy()


def _check_bounds(off, k, ok, cls, asc, frames):
    for s, e in frames:
        glo, ghi = _bounds(off, k, ok, cls, asc, s, e)
        elo, ehi = R.range_bounds(off, k, ok, cls, asc, s, e, loop=len(k) <= 1000)
        assert np.array_equal(glo, elo), (cls, asc, s, e)
        assert np.array_equal(ghi, ehi), (cls, asc, s, e)


FRAMES_INT = [(0, 0), (-1, 1), (-3, 0), (1, 3), (-3, -1), (None, 0), (0, None), (None, -1), (2, None), (-100, 100),
              (I64_MIN, I64_MAX), (I64_MIN, I64_MIN), (I64_MAX, I64_MAX), (-(2**62), 2**62)]
FRAMES_F64 = [(0, 0), (-0.25, 0.25), (-1.0, 0), (0.5, 2.0), (-2.0, -0.5), (None, 0), (0, None), (None, -0.25),
              (-1e308, 1e308), (1e308, 1e308), (-5e-324, 5e-324)]


@pytest.mark.parametrize("cls", ["I64", "U64", "F64"])
@pytest.mark.parametrize("ascending", [True, False])
@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 40 * TILE + 7])
def test_bounds_kernel_matches_oracle(cls, ascending, n):
    rng = np.random.default_rng(n + 3 * ascending + ord(cls[0]))
    frames = FRAMES_F64 if cls == "F64" else FRAMES_INT
    for shape in ("singletons", "zipf", "spanning"):
        off = _offsets(n, shape, rng)
        keys = _keys(n, cls, rng, spread=max(n // 8, 3))
        valid = rng.random(n) < (0.9 if shape != "spanning" else 1.0)  # spanning: no NULL key, no mask
        if len(off) > 3 and off[2] > off[1]:
            valid[off[1]:off[2]] = False  # an all-NULL segment
        k, ok = _sorted(off, keys, valid, cls, ascending)
        _check_bounds(off, k, ok, cls, ascending, frames)


def test_bounds_at_the_edges_of_the_key_types():
    off = np.array([0, 4, 8], dtype=np.int64)
    k = np.array([I64_MAX - 3, I64_MAX - 2, I64_MAX - 1, I64_MAX, I64_MIN, I64_MIN + 1, I64_MIN + 2, I64_MIN + 3])
    ok = np.ones(8, dtype=bool)
    for frame in [(1, 3), (-3, -1), (0, 0), (I64_MIN, I64_MAX)]:
        _check_bounds(off, k, ok, "I64", True, [frame])
        _check_bounds(off, k[::-1].copy(), ok, "I64", False, [frame])
    glo, ghi = _bounds(off, k, ok, "I64", True, 1, 3)
    assert ghi[3] < glo[3]  # INT64_MAX + 1 .. + 3 holds nothing: exact, not saturated
    u = np.array([0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 2, 2**64 - 1, 2**64 - 1], dtype=np.uint64).view(np.int64)
    off2 = np.array([0, 8], dtype=np.int64)
    for frame in [(1, 3), (-3, -1), (-1, 1), (I64_MIN, I64_MAX), (I64_MAX, I64_MAX), (0, 0)]:
        _check_bounds(off2, u, ok, "U64", True, [frame])
        _check_bounds(off2, u[::-1].copy(), ok, "U64", False, [frame])
    f = np.array([-np.inf, -1e308, -5e-324, -0.0, 0.0, 5e-324, 1e308, np.inf])
    for frame in [(0, 0), (-1e308, 1e308), (1e308, 1e308), (-7.0, 7.0), (-5e-324, 0)]:
        _check_bounds(off2, f, ok, "F64", True, [frame])
        _check_bounds(off2, f[::-1].copy(), ok, "F64", False, [frame])


def test_bounds_all_equal_all_null_and_large():
    rng = np.random.default_rng(9)
    n = 3_000_017
    off = np.array([0, n], dtype=np.int64)
    _check_bounds(off, np.full(n, 7, dtype=np.int64), np.ones(n, dtype=bool), "I64", True, [(-1, 1), (1, 2), (0, 0)])
    _check_bounds(off, np.zeros(n, dtype=np.int64), np.zeros(n, dtype=bool), "I64", False, [(-1, 1), (None, 0)])
    for shape in ("zipf", "spanning"):
        off = _offsets(n, shape, rng)
        k, ok = _sorted(off, _keys(n, "I64", rng, spread=n), rng.random(n) < 0.95, "I64", shape == "zipf")
        _check_bounds(off, k, ok, "I64", shape == "zipf", [(-40, 0), (-1, 1), (None, 0), (5, 900), (0, None)])


# ---- the aggregate kernel --------------------------------------------------------------------------
def _values(op, n, rng):
    if op == "SUM_F64":  # multiples of 2^-10 below 2^20: every partial sum is exact, so any order is bit-exact
        return (rng.integers(-(2**30), 2**30, n) * 2.0 ** -10).view(np.int64)
    if op.endswith("F64"):
        special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -1.5], dtype=np.float64)
        return np.where(rng.random(n) < 0.2, rng.choice(special, n), rng.standard_normal(n)).view(np.int64)
    return rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)


def _bounded(lo, hi, cols):
    spec = [(OPS[op], None if op == "COUNT" else torch.from_numpy(v).to(DEV),
             None if m is None else torch.from_numpy(m.astype(np.uint8)).to(DEV)) for op, v, m in cols]
    res = K.window_bounded(torch.from_numpy(lo).to(DEV), torch.from_numpy(hi).to(DEV), spec)
    return [(None if o is None else o.view(torch.int64).cpu().numpy(), c.cpu().numpy()) for o, c in res]


def _check_bounded(lo, hi, cols):
    for (op, v, m), (gv, gc) in zip(cols, _bounded(lo, hi, cols)):
        ev, ec = R.bounded_aggregate(None if op == "COUNT" else v, m, lo, hi, op, loop=False)
        assert np.array_equal(gc, ec), (op, m is not None)
        if op != "COUNT":
            assert np.array_equal(gv, ev), (op, m is not None)


@pytest.mark.parametrize("n", [0, 1, 2, 255, 256, 257, 5000, 100_003])
def test_bounded_kernel_on_arbitrary_bounds(n):
    rng = np.random.default_rng(n + 1)
    cols = [(op, _values(op, n, rng), m) for op in OPS for m in (None, rng.random(n) < 0.7)]  # 14: two batches
    pos = np.arange(n)
    lo = pos + rng.integers(-40, 10, n)
    hi = pos + rng.integers(-10, 40, n)
    wild = rng.random(n) < 0.05  # non-monotone, empty and out-of-range bounds
    lo[wild] = rng.integers(-2 * n - 5, 2 * n + 5, int(wild.sum()))
    hi[wild] = rng.integers(-2 * n - 5, 2 * n + 5, int(wild.sum()))
    if n > 4:
        lo[:2], hi[:2] = [I64_MIN, I64_MAX], [I64_MAX, I64_MIN]
        lo[2], hi[2] = -1, n  # one past each end: clamped
    _check_bounded(lo, hi, cols)


def test_bounded_against_the_loop_with_fsum():
    rng = np.random.default_rng(2)
    n = 3000
    pos = np.arange(n)
    lo, hi = pos - rng.integers(0, 300, n), pos + rng.integers(-5, 50, n)
    x = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).view(np.int64)
    m = rng.random(n) < 0.8
    (gv, gc), = _bounded(lo, hi, [("SUM_F64", x, m)])
    ev, ec = R.bounded_aggregate(x, m, lo, hi, "SUM_F64", loop=True)
    assert np.array_equal(gc, ec)
    g, e = gv.view(np.float64), ev.view(np.float64)
    xa = np.abs(np.where(m, x.view(np.float64), 0.0))
    ca = np.concatenate([[0.0], np.cumsum(xa)])
    mass = ca[np.clip(hi + 1, 0, n)] - ca[np.clip(lo, 0, n)]
    w = np.maximum(gc, 1)
    assert np.all(np.abs(g - e) <= (np.ceil(np.log2(w)) + 2) * 2.0 ** -52 * np.maximum(mass, 0) + 1e-300)


def test_a_huge_value_stays_in_its_frames_and_runs_repeat():
    n = 100_000
    v = np.ones(n)
    v[500] = 1e20
    pos = np.arange(n)
    lo, hi = pos - 6, pos
    cols = [("SUM_F64", v.view(np.int64), None)]
    (gv, _), = _bounded(lo, hi, cols)
    s = gv.view(np.float64)
    assert np.all(s[507:] == 7.0) and np.all(s[7:500] == 7.0) and np.all(s[500:507] > 1e19)
    rng = np.random.default_rng(4)
    x = rng.standard_normal(n).view(np.int64)
    lo2, hi2 = pos - rng.integers(0, 5000, n), pos + rng.integers(0, 5000, n)
    first = _bounded(lo2, hi2, [("SUM_F64", x, None)])[0][0]
    for _ in range(2):
        assert np.array_equal(_bounded(lo2, hi2, [("SUM_F64", x, None)])[0][0], first)


def test_one_segment_of_three_million_rows_up_to_the_current_peers():
    rng = np.random.default_rng(8)
    n = 3_000_017
    off = np.array([0, n], dtype=np.int64)
    k = np.sort(rng.integers(0, n // 3, n))
    ok = np.ones(n, dtype=bool)
    lo, hi = _bounds(off, k, ok, "I64", True, None, 0)
    elo, ehi = R.range_bounds(off, k, ok, "I64", True, None, 0)
    assert np.array_equal(lo, elo) and np.array_equal(hi, ehi)
    cols = [(op, _values(op, n, rng), rng.random(n) < 0.9) for op in ("SUM_F64", "SUM_I64", "MIN_F64", "MAX_I64")]
    cols.append(("COUNT", None, None))
    _check_bounded(lo, hi, cols)


# ---- whole maps ------------------------------------------------------------------------------------
def _maps_equal(got, exp, names):
    at = np.argsort(np.asarray(got.column("rid")))
    for c in names:
        g = [got.column(c)[int(i)].as_py() for i in at]
        e = exp[c]
        if c.startswith("sx") or c.startswith("ax"):
            for a, b in zip(g, e):
                assert (a is None) == (b is None), c
                if a is not None:
                    assert math.isclose(a, b, rel_tol=1e-9, abs_tol=1e-9), (c, a, b)
        else:
            assert g == e, c


def _range_cols(frame, tag):
    return [f.sum(col("v")).over(range=frame).alias(f"sv{tag}"), f.count(all_cols()).over(range=frame).alias(f"c{tag}"),
            f.max(col("x")).over(range=frame).alias(f"mx{tag}"), f.first(col("v")).over(range=frame).alias(f"fv{tag}"),
            f.last(col("x")).over(range=frame).alias(f"lx{tag}"), f.avg(col("x")).over(range=frame).alias(f"ax{tag}")]


PRESORT_TYPES = {
    "int8": (pa.int8(), lambda r, n: r.integers(-100, 100, n)),
    "int32": (pa.int32(), lambda r, n: r.integers(-50, 50, n)),
    "int64": (pa.int64(), lambda r, n: r.integers(-50, 50, n)),
    "uint16": (pa.uint16(), lambda r, n: r.integers(0, 60, n)),
    "uint64": (pa.uint64(), lambda r, n: r.integers(0, 60, n).astype(np.uint64) + np.uint64(2**63)),
    "float16": (pa.float16(), lambda r, n: (r.integers(-40, 40, n) / 4).astype(np.float16)),
    "float32": (pa.float32(), lambda r, n: (r.integers(-40, 40, n) / 4).astype(np.float32)),
    "float64": (pa.float64(), lambda r, n: np.where(r.random(n) < 0.05, np.inf, r.integers(-40, 40, n) / 4)),
    "date32": (pa.date32(), lambda r, n: r.integers(18000, 18060, n).astype(np.int32)),
    "date64": (pa.date64(), lambda r, n: r.integers(0, 40, n) * 86_400_000),
    "ts_s": (pa.timestamp("s"), lambda r, n: r.integers(0, 200, n) * 3600),
    "ts_us": (pa.timestamp("us"), lambda r, n: r.integers(0, 40, n) * 86_400_000_000 // 2),
    "ts_ns_tz": (pa.timestamp("ns", tz="UTC"), lambda r, n: r.integers(0, 40, n) * 3600 * 10**9 * 12),
    "duration_ms": (pa.duration("ms"), lambda r, n: r.integers(0, 100, n) * 1000),
    "time64_us": (pa.time64("us"), lambda r, n: r.integers(0, 100, n) * 1_000_000),
}
OFFSETS = {"int8": (-5, 0), "int32": (-3, 2), "int64": (1, 4), "uint16": (-4, -1), "uint64": (-3, 3),
           "float16": (-1.0, 0.5), "float32": (-0.75, 0), "float64": (-1, 1.5), "date32": (TD(days=-7), 0),
           "date64": (-3 * 86_400_000, 0), "ts_s": (TD(hours=-6), TD(hours=2)), "ts_us": (TD(days=-2), 0),
           "ts_ns_tz": (TD(hours=-36), 0), "duration_ms": (-5000, 5000), "time64_us": (TD(seconds=-10), 0)}


def _table(rng, n, tp, gen):
    t = pa.array(gen(rng, n), mask=rng.random(n) < 0.08).cast(tp) if not pa.types.is_temporal(tp) or \
        pa.types.is_date32(tp) else None
    if t is None:
        storage = pa.array(gen(rng, n).astype(np.int64), mask=rng.random(n) < 0.08)
        t = storage.view(tp) if not pa.types.is_date64(tp) else storage.cast(pa.date64())
    return pa.table({"rid": np.arange(n), "key": rng.integers(0, 12, n), "t": t,
                     "v": pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.1),
                     "x": pa.array(rng.standard_normal(n), mask=rng.random(n) < 0.1)})


def _run_map(tbl, cols, by, presort, algo="hash"):
    sch = Schema(tbl.schema)
    fields = [("rid", pa.int64())] + [(c.output_name, c.infer_type(sch) or pa.float64()) for c in cols]
    spec = PartitionSpec(by=by, algo=algo, **({"presort": presort} if presort else {}))
    return fa.transform(B200DataFrame(B200Table.from_arrow(tbl, DEV)), ColumnMap("rid", *cols),
                        schema=",".join(f"{n}:{type_to_expr(t)}" for n, t in fields), partition=spec, engine=_engine(),
                        as_fugue=True).as_arrow()


@pytest.mark.parametrize("name", list(PRESORT_TYPES))
@pytest.mark.parametrize("ascending", [True, False])
def test_transform_on_every_presort_type(name, ascending):
    rng = np.random.default_rng(len(name) * 31 + ascending)
    tp, gen = PRESORT_TYPES[name]
    tbl = _table(rng, 3000, tp, gen)
    cols = _range_cols(OFFSETS[name], "a") + _range_cols((None, 0), "b")
    presort = OrderedDict(t=ascending)
    got = _run_map(tbl, cols, ["key"], f"t {'asc' if ascending else 'desc'}")
    exp = R.window_map(tbl, ["key"], presort, [col("rid")] + cols)
    _maps_equal(got, exp, [c.output_name for c in cols])


@pytest.mark.parametrize("algo", ["hash", "even", "rand"])
def test_transform_mixes_range_rows_running_and_rank_nodes(algo):
    rng = np.random.default_rng(len(algo))
    tbl = _table(rng, 20_000, pa.int64(), lambda r, n: r.integers(0, 2000, n))
    cols = _range_cols((-30, 0), "a") + _range_cols((0, 0), "b") + _range_cols((-5, 10), "c") + [
        f.sum(col("v")).over(rows=(-3, 1)).alias("rw"), f.sum(col("v")).over(running=True).alias("run"),
        f.rank().alias("rk"), (col("v") - f.avg(col("x")).over(range=(-30, 0))).alias("ex")]
    got = _run_map(tbl, cols, ["key"], "t desc", algo)
    exp = R.window_map(tbl, ["key"], OrderedDict(t=False), [col("rid")] + cols)
    names = [c.output_name for c in cols]
    _maps_equal(got, exp, [c for c in names if c != "ex"])
    g = np.array([x if x is not None else np.nan for x in got.column("ex").to_pylist()], dtype=float)
    e = np.array([x if x is not None else np.nan for x in exp["ex"]], dtype=float)[np.argsort(np.argsort(
        np.asarray(got.column("rid"))))]
    assert np.allclose(g, e, rtol=1e-9, atol=1e-9, equal_nan=True)


def test_peer_frames_with_several_or_no_presort_columns():
    rng = np.random.default_rng(12)
    tbl = _table(rng, 4000, pa.int64(), lambda r, n: r.integers(0, 20, n)).append_column(
        "u", pa.array(rng.integers(0, 3, 4000)))
    cols = _range_cols((None, 0), "a") + _range_cols((0, 0), "b") + _range_cols((0, None), "c")
    got = _run_map(tbl, cols, ["key"], "t desc, u")
    exp = R.window_map(tbl, ["key"], OrderedDict(t=False, u=True), [col("rid")] + cols)
    _maps_equal(got, exp, [c.output_name for c in cols])
    got = _run_map(tbl, cols, ["key"], None)
    exp = R.window_map(tbl, ["key"], OrderedDict(), [col("rid")] + cols)
    _maps_equal(got, exp, [c.output_name for c in cols])


def test_evaluation_time_errors():
    rng = np.random.default_rng(1)
    tbl = _table(rng, 200, pa.int64(), lambda r, n: r.integers(0, 20, n)).append_column(
        "s", pa.array(["a", "b"] * 100)).append_column("b", pa.array([True, False] * 100)).append_column(
        "d", pa.array(np.arange(200, dtype=np.int32)).view(pa.date32())).append_column(
        "fl", pa.array(rng.standard_normal(200)))
    bad = [((-1, 0), None), ((-1, 0), "t, v"), ((-1, 0), "s"), ((-1, 0), "b"), ((-1.5, 0), "t"),
           ((TD(days=-1), 0), "t"), ((TD(days=-1), 0), "fl"), ((TD(hours=-36), 0), "d"), ((0.5, 1.0), "d"),
           ((-(2**63) - 1, 0), "t")]
    for frame, presort in bad:
        with pytest.raises(ValueError):
            _run_map(tbl, [f.sum(col("v")).over(range=frame).alias("s1")], ["key"], presort)
