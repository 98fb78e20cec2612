"""Every aggregate head through every route that runs it, against the exact reference (tests/_aggregate_reference.py),
at the edge values of every column type.

``fugue_b200/aggregates.py`` defines each function once; up to seven routes run that definition with different
kernels:

* ``hash`` / ``hash_partitioned`` - ``engine.aggregate`` of plain ``FUNC(col)``: K6 ``fb_groupby_u64`` over the
  whole table, or (``K.GROUPBY_PARTITION_MIN_ROWS`` lowered) its lean / region kernels;
* ``sorted`` - the same call with a percentile added: a stable sort, then the K9 scans and K10;
* ``select`` - ``engine.select`` with a HAVING clause: the device evaluator around K6 (or the sorted route);
* ``whole`` / ``running`` - ``f.x(c).over()`` / ``over(running=True)`` in a ColumnMap: the K9 segmented scans;
* ``rows_tile`` / ``rows_combine`` - ``over(rows=(-511, 511))`` on groups of at most 512 rows (the one-pass tile
  kernel) and ``over(rows=(-3000, 3000))`` on a longer table (the prefix / suffix scans and their combine);
* ``range`` - ``over(range=(-R, R))`` on an integer presort column whose span in every group is below R.

Which routes a function takes follows ``AGGREGATES[fn].frames``; the frames chosen cover every group, so every row
must hold the group's aggregate.  A spy on the C entry points checks which kernels ran.

Integer results, COUNT, MIN, MAX, FIRST, LAST, PERCENTILE_DISC / _CONT and REGR_COUNT are compared bit for bit,
with the result type of ``column.result_type``; a float SUM / AVG within ``(m - 1) 2^-52 sum |x|`` of the exact value
(plus one rounding of the quotient for AVG); the variances, shape statistics and pair functions within the bounds of
tests/test_moments_gpu.py, oracle/shape_moments.py and tests/test_comoments_gpu.py.
"""
import functools
import math
from collections import OrderedDict
from fractions import Fraction
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import _aggregate_reference as R  # noqa: E402
import _frame_oracle as FO  # noqa: E402
import _range_oracle as RO  # noqa: E402
import test_comoments_gpu as TC  # noqa: E402 - the pair functions' bounds
import test_moments_gpu as TM  # noqa: E402 - the variances' bounds
from fugue_b200 import _lib  # noqa: E402
from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import AGGREGATES, SelectColumns, all_cols, col, functions as ff, result_type  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.schema import Schema  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402
from oracle import groupby as og  # noqa: E402
from oracle import shape_moments as OS  # noqa: E402

DEV = torch.device("cuda", 0)
DBL_MAX = 1.7976931348623157e308
RANGE = 8000          # above the span of the presort column p in every group
LONG = 2500           # rows of the group longer than a K9 tile (2048) and K10's one-pass tile
TILE_GROUP_MAX = 512  # groups the tile-path frame (-511, 511) covers whole

# ---- the table ------------------------------------------------------------------------------------
TYPES = OrderedDict([
    ("i8", pa.int8()), ("i16", pa.int16()), ("i32", pa.int32()), ("i64", pa.int64()),
    ("u8", pa.uint8()), ("u16", pa.uint16()), ("u32", pa.uint32()), ("u64", pa.uint64()),
    ("f16", pa.float16()), ("f32", pa.float32()), ("f64", pa.float64()), ("b", pa.bool_()),
    ("d32", pa.date32()), ("d64", pa.date64()), ("ts_s", pa.timestamp("s")), ("ts_ms", pa.timestamp("ms")),
    ("ts_us", pa.timestamp("us")), ("ts_ns", pa.timestamp("ns")), ("ts_tz", pa.timestamp("ms", "Asia/Kolkata")),
    ("s", pa.string()),
])
_NP = {"i8": np.int8, "i16": np.int16, "i32": np.int32, "i64": np.int64, "u8": np.uint8, "u16": np.uint16,
       "u32": np.uint32, "u64": np.uint64}
# quiet NaNs of both signs, and NaNs with payloads (signalling ones among them): widen / narrow keep every bit
_F16_NAN = np.array([0x7E00, 0xFE00, 0x7C01, 0xFD55, 0x7FFF, 0xFE01], np.uint16).view(np.float16)
_F32_NAN = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFA00005, 0x7FFFFFFF, 0xFFC00123], np.uint32).view(np.float32)
_F64_NAN = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001],
                    np.uint64).view(np.float64)
_FLOAT_EDGES = {  # (finite edges, non-finite edges)
    "f16": (np.array([65504, -65504, 2.0 ** -24, -(2.0 ** -24), -0.0, 0.0], np.float16),
            np.concatenate([np.array([np.inf, -np.inf], np.float16), _F16_NAN])),
    "f32": (np.array([3.4028235e38, -3.4028235e38, 2.0 ** -149, -0.0], np.float32),
            np.concatenate([np.array([np.inf, -np.inf], np.float32), _F32_NAN])),
    # the subnormals go with the specials (a large group holding one costs the exact shape reference 2^4296-bit
    # fractions); the small all-finite group 0 gives the moments subnormal input
    "f64": (np.array([-0.0, 0.0]), np.concatenate([[np.inf, -np.inf, 5e-324, -5e-324], _F64_NAN])),
}
_STRINGS = np.array(["", "a", "Z", "é", "日本語", "🙂", "ab", "é🙂", "zz"], dtype=object)
_TEMPORAL = {"d32": (40_000, [-719_162, 2_932_896]), "d64": (40_000, [-719_162, 2_932_896]),
             "ts_s": (2**40, [-(2**40), 2**40]), "ts_ms": (2**50, [-(2**52), 2**52]),
             "ts_us": (2**58, [-(2**60), 2**60]), "ts_ns": (2**62, [-(2**62), 2**62]),
             "ts_tz": (2**50, [-(2**52), 2**52])}


def _values(name: str, kind: str, special: bool, rng: np.random.Generator, n: int) -> Tuple[np.ndarray, np.ndarray]:
    """(values, validity) of column ``name`` for a group of ``n`` rows of ``kind``."""
    valid = np.ones(n, bool) if kind != "allnull" else np.zeros(n, bool)
    if kind == "mixed":
        valid = rng.random(n) > 0.15
    edge = rng.random(n) < 0.3
    if name in _NP:
        t = _NP[name]
        info = np.iinfo(t)
        v = rng.integers(info.min, info.max, n, dtype=t, endpoint=True)
        v[edge] = rng.choice(np.array([info.min, info.max], t), int(edge.sum()))
        if name == "u64":  # values at and just above 2^63
            top = rng.random(n) < 0.2
            v[top] = np.uint64(2**63) + rng.integers(0, 5, int(top.sum())).astype(np.uint64)
        if kind == "negative" and info.min < 0:
            v = np.where(v > 0, -v, v).astype(t)
        return (np.zeros(n, t) if kind == "zeros" else v), valid
    if name in _FLOAT_EDGES:
        dt = {"f16": np.float16, "f32": np.float32, "f64": np.float64}[name]
        scale = {"f16": 3, "f32": 30, "f64": 30}[name]
        x = rng.standard_normal(n) * 10.0 ** rng.uniform(-scale, scale, n)
        if name == "f16":
            x = np.clip(x, -60000, 60000)
        x = x.astype(dt)
        fin, nonfin = _FLOAT_EDGES[name]
        pool = np.concatenate([fin, nonfin]) if special else fin
        x[edge] = rng.choice(pool, int(edge.sum()))
        if kind == "nan":
            x = rng.choice(_F16_NAN if name == "f16" else _F32_NAN if name == "f32" else _F64_NAN, n).astype(dt)
        elif kind == "zeros":
            x = rng.choice(np.array([0.0, -0.0], dt), n)
        elif kind == "overflow" and name == "f64":  # DBL_MAX pairs: the sum overflows in every order
            x = np.resize(np.array([DBL_MAX, DBL_MAX, -1.0, 2.0]), n)
        elif kind == "negative":  # every sign bit set: MAX in totalOrder is the smallest magnitude, -0.0 or -NaN
            x = -np.abs(x)
        elif kind == "subnormal" and name == "f64":  # finite, a third of it subnormal: the moments see them too
            x[::3] = rng.choice(np.array([5e-324, -5e-324, 1e-310, -2.5e-320]), len(x[::3]))
        return x, valid
    if name == "b":
        return (rng.random(n) < 0.5) & (kind != "zeros"), valid
    if name == "s":
        return (np.full(n, "", object) if kind == "zeros" else rng.choice(_STRINGS, n)), valid
    span, edges = _TEMPORAL[name]
    v = rng.integers(-span, span, n)
    v[edge] = rng.choice(np.array(edges), int(edge.sum()))
    if kind == "negative":
        v = -np.abs(v)
    if name == "d64":
        v = v * 86_400_000
    return (np.zeros(n, np.int64) if kind == "zeros" else v), valid


def _arrow(name: str, v: np.ndarray, valid: np.ndarray) -> pa.Array:
    tp = TYPES[name]
    if name == "s":
        return pa.array([x if ok else None for x, ok in zip(v.tolist(), valid.tolist())], type=pa.string())
    if name in _TEMPORAL:
        return pa.array(v.astype(np.int32 if name == "d32" else np.int64), mask=~valid).cast(tp)
    return pa.array(v, mask=~valid, type=tp)


class Data:
    """One table of several key groups (rows interleaved), its groups in input row order and its device frame."""

    def __init__(self, tbl: pa.Table):
        self.tbl = tbl
        self.n = tbl.num_rows
        keys = R.canonical(tbl.column("g"))
        self.groups: Dict[Any, List[int]] = {}
        for i, k in enumerate(keys):
            self.groups.setdefault(k, []).append(i)
        self.cols = {nm: R.canonical(tbl.column(nm)) for nm in list(TYPES) + ["yf"]}
        self.o = tbl.column("o").to_numpy()
        self.row_of = {r: i for i, r in enumerate(tbl.column("rid").to_pylist())}  # a result's rid -> our row

    @functools.cached_property
    def df(self) -> B200DataFrame:
        return B200DataFrame(B200Table.from_arrow(self.tbl, DEV))

    def values(self, name: str, key: Any) -> List[Any]:
        c = self.cols[name]
        return [c[i] for i in self.groups[key]]


@functools.lru_cache(maxsize=None)
def full() -> Data:
    rng = np.random.default_rng(2024)
    spec = [(None, "mixed", 40), (1, "allnull", 6), (2, "mixed", 1), (3, "nan", 5), (4, "zeros", 6),
            (5, "overflow", 4), (6, "mixed", LONG), (7, "negative", 30), (8, "negative", 30),
             (0, "subnormal", 12)]
    spec += [(10 + i, "mixed", int(rng.integers(1, 501))) for i in range(40)]
    parts: Dict[str, List[Any]] = {nm: [] for nm in TYPES}
    gkeys: List[Any] = []
    yf: List[Any] = []
    for key, kind, n in spec:
        special = key is None or (key % 2 == 1)
        for nm in TYPES:
            parts[nm].append(_values(nm, kind, special, rng, n))
        gkeys += [key] * n
        y = rng.standard_normal(n)
        yf += [None if r < 0.1 else float(x) for x, r in zip(y, rng.random(n))]
    order = rng.permutation(len(gkeys))  # interleave the groups
    cols: Dict[str, Any] = {}
    g = np.array([-1 if k is None else k for k in gkeys], np.int64)[order]
    gnull = np.array([k is None for k in gkeys])[order]
    cols["g"] = pa.array(g, mask=gnull)
    cols["rid"] = pa.array(np.arange(len(order), dtype=np.int64))
    # o: the position in the group in input row order; p: a non-decreasing presort key (ties allowed) in that order
    o, p = np.zeros(len(order), np.int64), np.zeros(len(order), np.int64)
    seen: Dict[Any, Tuple[int, int]] = {}
    gaps = rng.integers(0, 4, len(order))
    for i, (k, nul) in enumerate(zip(g.tolist(), gnull.tolist())):
        kk = None if nul else k
        c, last = seen.get(kk, (0, 0))
        o[i], p[i] = c, last + (gaps[i] if c else 0)
        seen[kk] = (c + 1, p[i])
    cols["o"], cols["p"] = pa.array(o), pa.array(p)
    for nm in TYPES:
        v = np.concatenate([x for x, _ in parts[nm]])[order]
        m = np.concatenate([m for _, m in parts[nm]])[order]
        cols[nm] = _arrow(nm, v, m)
    cols["yf"] = pa.array([yf[i] for i in order], type=pa.float64())
    return Data(pa.table(cols))


@functools.lru_cache(maxsize=None)
def small() -> Data:
    """The groups of at most ``TILE_GROUP_MAX`` rows."""
    d = full()
    keep = np.zeros(d.n, bool)
    for rows in d.groups.values():
        if len(rows) <= TILE_GROUP_MAX:
            keep[rows] = True
    return Data(d.tbl.filter(pa.array(keep)))


# ---- the launch spy -------------------------------------------------------------------------------
SCAN_OF = {"basic": "fb_segmented_scan", "pick": "fb_segmented_scan", "variance": "fb_segmented_moments",
           "shape": "fb_segmented_shape_moments", "bivariate": "fb_segmented_comoments",
           "percentile": "fb_segmented_quantile"}
ENTRIES = ("fb_groupby_u64", "fb_segmented_scan", "fb_segmented_moments", "fb_segmented_shape_moments",
           "fb_segmented_comoments", "fb_window_frame", "fb_window_bounded", "fb_segmented_quantile")


class Launches:
    """(entry point, detail) of every call of the C entry points of the aggregate kernels: the K6 path
    (``generic``, ``lean<N>``, ``region``, ``batched``) with its row count, and whether ``fb_window_frame`` took
    its one-pass tile kernel."""

    def __init__(self, monkeypatch: Any):
        lib = _lib.load()
        self.calls: List[Tuple[str, Any]] = []
        for nm in ENTRIES:
            monkeypatch.setattr(lib, nm, self._spy(nm, getattr(lib, nm)))

    def _spy(self, nm: str, real: Any) -> Any:
        def spy(*a: Any) -> int:
            detail = None
            if nm == "fb_groupby_u64":
                naggs, parts, batched = a[5], a[10], bool(a[13])
                path = "generic" if parts == 0 else "batched" if batched else \
                    f"lean{naggs}" if 1 <= naggs <= 4 else "region"
                detail = (a[2], path)
            elif nm == "fb_window_frame":
                s, e, flags = a[5], a[6], a[7]
                detail = "tile" if flags == 0 and e - s + 1 <= K.FRAME_TILE_MAX_WIDTH else "combine"
            self.calls.append((nm, detail))
            return real(*a)

        return spy

    def names(self) -> set:
        return {c[0] for c in self.calls}

    def details(self, nm: str) -> List[Any]:
        return [d for c, d in self.calls if c == nm]


@pytest.fixture
def launches(monkeypatch):
    return Launches(monkeypatch)


@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


# ---- routes ---------------------------------------------------------------------------------------
FAMILIES: Dict[str, List[str]] = {}
for _fn, _a in AGGREGATES.items():
    FAMILIES.setdefault(_a.family, []).append(_fn)
K6_ROUTES = ("hash", "hash_partitioned", "select")
WINDOW_OVER = {"whole": {}, "running": {"running": True}, "rows_tile": {"rows": (-511, 511)},
               "rows_combine": {"rows": (-3000, 3000)}, "range": {"range": (-RANGE, RANGE)}}
ROUTES = ["hash", "hash_partitioned", "sorted", "select"] + list(WINDOW_OVER)
QS = {"PERCENTILE_DISC": (0.0, 0.5, 1.0), "PERCENTILE_CONT": (0.25, 1.0)}


def routes_of(fn: str) -> List[str]:
    frames = AGGREGATES[fn].frames
    if frames == "none":  # a percentile: the sorted route in aggregate and select, the whole partition
        return ["sorted", "select", "whole"]
    return ROUTES if frames == "any" else [r for r in ROUTES if not r.startswith(("rows", "range"))]


def expr(fn: str, c: str, q: Optional[float] = None) -> Any:
    b = getattr(ff, fn.lower())
    if AGGREGATES[fn].family == "bivariate":  # x is c, y is yf: CORR(x, y), REGR_*(y, x)
        return b(col("yf"), col(c)) if fn.startswith("REGR_") else b(col(c), col("yf"))
    return b(col(c)) if q is None else b(col(c), q)


def data_of(route: str) -> Data:
    return small() if route == "rows_tile" else full()


def run(route: str, d: Data, specs: List[Tuple[str, str, str, Optional[float]]], engine: Any,
        monkeypatch: Any) -> Dict[str, Dict[Any, List[Any]]]:
    """Run the aggregates ``specs`` = (output name, function, column, q) through ``route``: per output, per group
    key, its results (one per group; one per row for a window, the last row's for a running window).  Checks
    the result type against ``column.result_type``."""
    if route == "hash_partitioned":
        monkeypatch.setattr(K, "GROUPBY_PARTITION_MIN_ROWS", 64)
    aggs = [expr(fn, c, q).alias(nm) for nm, fn, c, q in specs]
    if route in ("hash", "hash_partitioned", "sorted"):
        if route == "sorted":
            aggs.append(ff.percentile_disc(col("u8"), 0.5).alias("__pd"))
        res = engine.aggregate(d.df, PartitionSpec(by="g"), aggs).as_arrow()
    elif route == "select":
        res = engine.select(d.df, SelectColumns(col("g"), *aggs), having=ff.count(all_cols()) >= 0).as_arrow()
    else:
        over = WINDOW_OVER[route]
        cols = [expr(fn, c, q).over(**over).alias(nm) for nm, fn, c, q in specs]
        schema = Schema([pa.field("g", pa.int64()), pa.field("rid", pa.int64())]
                        + [pa.field(nm, result_type(fn, TYPES.get(c))) for nm, fn, c, q in specs])
        res = fa.transform(d.df, ColumnMap(col("g"), col("rid"), *cols), schema=schema,
                           partition=PartitionSpec(by="g", presort="p asc"), engine=engine,
                           as_fugue=True).as_arrow()
    for nm, fn, c, q in specs:
        assert res.schema.field(nm).type == result_type(fn, TYPES[c]), (route, nm, res.schema.field(nm).type)
    keys = R.canonical(res.column("g"))
    out: Dict[str, Dict[Any, List[Any]]] = {}
    if route in ("hash", "hash_partitioned", "sorted", "select"):
        assert len(keys) == len(set(keys)) == len(d.groups), (route, len(keys), len(d.groups))
        for nm, *_ in specs:
            out[nm] = {k: [v] for k, v in zip(keys, R.canonical(res.column(nm)))}
        return out
    rows = [d.row_of[r] for r in res.column("rid").to_pylist()]
    assert sorted(rows) == list(range(d.n))
    take = np.ones(len(rows), bool)
    if route == "running":  # the last row of every group holds the group's aggregate
        last: Dict[Any, Tuple[int, int]] = {}
        for i, (k, r) in enumerate(zip(keys, rows)):
            if k not in last or d.o[r] > last[k][0]:
                last[k] = (int(d.o[r]), i)
        take[:] = False
        take[[i for _, i in last.values()]] = True
    for nm, *_ in specs:
        vals = R.canonical(res.column(nm))
        per: Dict[Any, List[Any]] = {}
        for k, v, t in zip(keys, vals, take.tolist()):
            if t:
                per.setdefault(k, []).append(v)
        out[nm] = per
    return out


def kernels_ran(route: str, family: str, launches: Launches, d: Data) -> None:
    names = launches.names()
    scan = SCAN_OF[family]
    if route in K6_ROUTES and family != "percentile":
        assert "fb_groupby_u64" in names, (route, names)
        n_rows, path = launches.details("fb_groupby_u64")[-1]
        assert n_rows == d.n
        if route == "hash":
            assert path == "generic" and not names & set(SCAN_OF.values()), (path, names)
        elif route == "hash_partitioned":
            assert path in ("lean1", "lean2", "lean3", "lean4", "region") and not names & set(SCAN_OF.values())
    elif route in ("sorted", "select"):
        assert {"fb_segmented_quantile", scan} <= names, (route, names)
    elif route in ("whole", "running"):
        assert scan in names, (route, names)
    elif route == "range":
        assert "fb_window_bounded" in names, names
    else:
        assert launches.details("fb_window_frame") and \
            set(launches.details("fb_window_frame")) == {route.split("_")[1]}, launches.calls


# ---- comparison -----------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _reference(d: Data, c: str, key: Any, fn: str, q: Optional[float]) -> Any:
    ys = d.values("yf", key) if AGGREGATES[fn].family == "bivariate" else None
    return R.aggregate(fn, TYPES[c], d.values(c, key), q=q, ys=ys)


def _too_big(vals: List[Any]) -> bool:
    return any(isinstance(v, float) and math.isfinite(v) and abs(v) >= 2.0 ** 255 for v in vals)


def same(a: Any, b: Any) -> bool:
    if isinstance(a, float) and isinstance(b, float):
        return og.bits_of(a) == og.bits_of(b)
    return a == b and type(a) is type(b)


def _present(d: Data, c: str, key: Any) -> List[float]:
    return [float(v) for v in d.values(c, key) if v is not None]


@functools.lru_cache(maxsize=None)
def _variance_parts(d: Data, c: str, key: Any) -> Tuple[int, float, float]:
    """(m, exact M2, sum x^2) of a group's finite values, rounded once: the inputs of ``TM.m2_tol``."""
    vals = _present(d, c, key)
    return len(vals), float(R.OM.exact_m2(vals)), float(sum(Fraction(x) ** 2 for x in vals))


def check_variance(fn: str, got: Optional[float], want: Optional[float], d: Data, c: str, key: Any,
                   scan: bool) -> None:
    """``TM.check_result`` with the group's exact sums computed once for all routes and functions."""
    if want is None or math.isnan(want):
        assert (got is None) if want is None else math.isnan(got), (fn, c, key, got, want)
        return
    m, ex, sx2 = _variance_parts(d, c, key)
    tol_m2 = 4 * m * TM.U * math.sqrt(sx2 * ex) if scan else 2 * ((m + 2) * TM.U * ex + (m * TM.U) ** 2 * sx2)
    div = m - 1 if fn.endswith("_SAMP") else m
    var = ex / div
    tol = tol_m2 / div + 2 * TM.U * var
    g = got * got if fn.startswith("STDDEV") else got
    assert abs(g - var) <= tol + (4 * TM.U * var if fn.startswith("STDDEV") else 0), (fn, c, key, got, want)


@functools.lru_cache(maxsize=None)
def _pair_errors(d: Data, c: str, key: Any, scan: bool) -> Tuple[List[Tuple[float, float]], Any]:
    """The pair rows of x = column ``c``, y = yf in a group, and ``TC.errors`` of them (None where the float64
    sums of the pair overflow)."""
    pairs = R.OC.pair_rows([None if v is None else float(v) for v in d.values(c, key)], d.values("yf", key))
    if R._too_big([v for p in pairs for v in p], 2.0 ** 511):
        return pairs, None
    return pairs, TC.errors(pairs, scan)


def check_one_square(fn: str, got: Optional[float], d: Data, c: str, key: Any, scan: bool) -> None:
    """REGR_SXX / REGR_SYY of pair rows whose squares overflow on one side: each reads one side only.  Sxx (Syy) of
    the side that overflows is not finite, of the other side within the variance bound."""
    pairs, _ = _pair_errors(d, c, key, scan)
    side = [p[0 if fn == "REGR_SXX" else 1] for p in pairs]
    if R._too_big(side, 2.0 ** 511):
        assert got is not None and not math.isfinite(got), (fn, c, key, got)
    else:
        assert abs(got - float(R.OM.exact_m2(side))) <= TM.m2_tol(side, scan), (fn, c, key, got)


def check_float_sum(fn: str, got: Optional[float], want: Optional[float], vals: List[Any], where: Tuple) -> None:
    """A float SUM or AVG of ``vals``: NULL, NaN and the infinities as the reference has them, a finite result within
    ``(m - 1) 2^-52 sum |x|`` of it (plus one rounding of the quotient for an AVG)."""
    if want is None or got is None:
        assert want is None and got is None, where
        return
    if math.isnan(want) or math.isinf(want):
        assert same(got, want) or (math.isnan(want) and math.isnan(got)), where
        return
    bound = R.sum_bound(vals)
    if fn == "AVG":
        bound = bound / len([v for v in vals if v is not None]) + 2.0 ** -52 * abs(want)
    assert not math.isnan(got) and abs(got - want) <= bound, where + (bound,)


@functools.lru_cache(maxsize=None)
def _central_sums(d: Data, c: str, key: Any) -> Any:
    return OS.central_sums(_present(d, c, key))


@functools.lru_cache(maxsize=None)
def _shape_bound(d: Data, c: str, key: Any, fn: str, kind: str) -> float:
    return OS.result_bound(fn, _present(d, c, key), kind)


def check(fn: str, c: str, route: str, got: Any, d: Data, key: Any, q: Optional[float]) -> None:
    tp = TYPES[c]
    vals = d.values(c, key)
    family = AGGREGATES[fn].family
    scan = route not in K6_ROUTES
    if fn in ("REGR_AVGX", "REGR_AVGY"):  # the averages follow AVG (DESIGN §7k) on every route
        side = [p[0 if fn == "REGR_AVGX" else 1] for p in _pair_errors(d, c, key, scan)[0]]
        want = _reference(d, c, key, fn, None)
        check_float_sum("AVG", got, want, side, (fn, c, route, key, got, want))
        return
    if family == "shape":  # the reference's value, from central sums computed once per group
        want = R.aggregate(fn, tp, vals) if _too_big(vals) else OS.finish(fn, _central_sums(d, c, key))
    elif family == "bivariate":  # the reference's value, from the exact state of the pair rows computed once
        pairs, pre = _pair_errors(d, c, key, scan)
        want = len(pairs) if fn == "REGR_COUNT" else R.OVERFLOW if pre is None else R.OC.result_of_state(fn, pre[0])
    else:
        want = _reference(d, c, key, fn, q)
    where = (fn, c, route, key, got, want)
    if want is R.OVERFLOW and fn in ("REGR_SXX", "REGR_SYY"):
        check_one_square(fn, got, d, c, key, scan)
        return
    if want is R.OVERFLOW:  # beyond the float64 power sums of every algorithm: no finite answer
        assert got is not None and not math.isfinite(got), where
        return
    if fn == "REGR_COUNT":
        assert same(got, want), where
        return
    if family == "variance":
        check_variance(fn, got, want, d, c, key, scan)
        return
    if family == "bivariate":
        pairs, pre = _pair_errors(d, c, key, scan)
        TC.check(fn, got, pairs, scan, pre)
        return
    if fn in ("SUM", "AVG") and pa.types.is_floating(result_type(fn, tp)):
        check_float_sum(fn, got, want, vals, where)
        return
    if want is None or got is None:
        assert want is None and got is None, where
        return
    if family == "shape":
        if math.isnan(want):
            assert math.isnan(got), where
        else:
            bound = _shape_bound(d, c, key, fn, "scan" if scan else "hash")
            assert abs(got - want) <= bound, where + (bound,)
        return
    assert same(got, want), where


def columns_for(fn: str) -> List[str]:
    return [c for c in TYPES if not R.rejects(fn, TYPES[c])]


CASES = [(route, fam) for fam, fns in FAMILIES.items() for route in ROUTES if any(route in routes_of(f) for f in fns)]


@pytest.mark.parametrize("route,family", CASES, ids=[f"{r}-{f}" for r, f in CASES])
def test_every_function_on_every_type_matches_the_reference(route, family, engine, monkeypatch, launches):
    d = data_of(route)
    fns = [f for f in FAMILIES[family] if route in routes_of(f)]
    cols = sorted({c for f in fns for c in columns_for(f)}, key=list(TYPES).index)
    assert cols
    for c in cols:
        specs = [(f"{f}@{q}" if q is not None else f, f, c, q) for f in fns if c in columns_for(f)
                 for q in QS.get(f, (None,))]
        launches.calls.clear()
        got = run(route, d, specs, engine, monkeypatch)
        kernels_ran(route, family, launches, d)
        for nm, fn, _, q in specs:
            assert set(got[nm]) == set(d.groups), (nm, route)
            for key, vs in got[nm].items():
                if AGGREGATES[fn].family in ("variance", "shape", "bivariate"):  # one value repeated on every row
                    assert all(same(v, vs[0]) or (v != v and vs[0] != vs[0]) for v in vs), (fn, c, route, key)
                # each distinct result of the group's rows once (a frame's rows may round a float sum apart)
                for v in {(type(v), og.bits_of(v) if isinstance(v, float) else v): v for v in vs}.values():
                    check(fn, c, route, v, d, key, q)


REJECT_FNS = ["VAR_POP", "STDDEV_SAMP", "KURTOSIS", "SKEWNESS_POP", "CORR", "REGR_SXY", "PERCENTILE_CONT", "SUM",
              "AVG"]


@pytest.mark.parametrize("fn", REJECT_FNS)
def test_a_rejected_argument_type_raises_the_same_on_every_route(fn, engine, monkeypatch):
    """The variances, shape statistics, pair functions and PERCENTILE_CONT refuse booleans, dates, timestamps and
    strings, SUM and AVG refuse strings - on every route with the same exception.  SUM and AVG of a bool, a date or
    a timestamp are computed (an int64 / float64 of the stored values); the matrix above compares them route by
    route."""
    rejected = [c for c in TYPES if R.rejects(fn, TYPES[c])]
    assert rejected
    for c in rejected:
        raised = {}
        for route in routes_of(fn):
            with pytest.raises(Exception) as e:
                run(route, data_of(route), [("r", fn, c, 0.5 if fn in QS else None)], engine, monkeypatch)
            raised[route] = type(e.value)
        assert set(raised.values()) == {NotImplementedError}, (fn, c, raised)


# ---- clipped frames, row by row -------------------------------------------------------------------
FRAME_GROUPS = [None, 0, 1, 2, 3, 4, 5, 7, 8, 10, 11]


@functools.lru_cache(maxsize=None)
def frame_data() -> Data:
    d = full()
    keep = np.zeros(d.n, bool)
    for k in FRAME_GROUPS:
        keep[d.groups[k]] = True
    return Data(d.tbl.filter(pa.array(keep)))


@pytest.mark.parametrize("frame", [("rows", (-3, 2)), ("rows", (1, 4)), ("range", (-2, 3)), ("range", (-5, -1))],
                         ids=lambda f: f"{f[0]}{f[1]}")
def test_clipped_frames_row_by_row(frame, engine, monkeypatch, launches):
    """Frames that do not cover their group, on every edge-value column: each row against the reference over the
    rows of its frame, which ``_frame_oracle.frame_bounds`` / ``_range_oracle.range_bounds`` give."""
    d = frame_data()
    kind, (s, e) = frame
    # the rows in presort order (key, then p; ties of p in input row order, as p follows it)
    keys = list(d.groups)
    order = [r for k in keys for r in d.groups[k]]
    offsets = np.cumsum([0] + [len(d.groups[k]) for k in keys]).astype(np.int64)
    if kind == "rows":
        lo, hi = FO.frame_bounds(offsets, s, e)
    else:
        p = d.tbl.column("p").to_numpy()[order]
        lo, hi = RO.range_bounds(offsets, p, None, "I64", True, s, e)
    frame_of = {order[i]: [order[j] for j in range(lo[i], hi[i] + 1)] for i in range(len(order))}
    for c in TYPES:
        fns = [f for f in FAMILIES["basic"] + FAMILIES["pick"] if not R.rejects(f, TYPES[c])]
        specs = [(f, f, c, None) for f in fns]
        aggs = [expr(f, c).over(**{kind: (s, e)}).alias(f) for f in fns]
        schema = Schema([pa.field("rid", pa.int64())] + [pa.field(f, result_type(f, TYPES[c])) for f in fns])
        launches.calls.clear()
        res = fa.transform(d.df, ColumnMap(col("rid"), *aggs), schema=schema,
                           partition=PartitionSpec(by="g", presort="p asc"), engine=engine, as_fugue=True).as_arrow()
        assert ("fb_window_frame" if kind == "rows" else "fb_window_bounded") in launches.names()
        rid = [d.row_of[r] for r in res.column("rid").to_pylist()]
        for nm, fn, _, _ in specs:
            assert res.schema.field(nm).type == result_type(fn, TYPES[c])
            col_ = d.cols[c]
            for r, got in zip(rid, R.canonical(res.column(nm))):
                vals = [col_[j] for j in frame_of[r]]
                want = R.aggregate(fn, TYPES[c], vals)
                where = (fn, c, frame, r, got, want)
                if fn in ("SUM", "AVG") and pa.types.is_floating(result_type(fn, TYPES[c])):
                    check_float_sum(fn, got, want, vals, where)
                elif want is None or got is None:
                    assert want is None and got is None, where
                else:
                    assert same(got, want), where


# ---- documented divergences -----------------------------------------------------------------------
def test_uint64_at_and_above_2_63_min_is_its_int64_pattern_but_percentile_disc_is_unsigned(engine, launches):
    """DESIGN §7e: a uint64 value >= 2^63 stays its int64 bit pattern for MIN / MAX (and SUM, AVG, the variances),
    while the quantile kernel orders uint64 as unsigned: PERCENTILE_DISC(0) is not MIN on such a column."""
    t = pa.table({"g": pa.array([0, 0, 0], pa.int64()), "v": pa.array([1, 2**63, 3], pa.uint64()),
                  "p": pa.array([0, 1, 2], pa.int64())})
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    res = engine.aggregate(df, PartitionSpec(by="g"), [ff.min(col("v")).alias("mn"), ff.max(col("v")).alias("mx")])
    assert "fb_groupby_u64" in launches.names()
    row = res.as_arrow().to_pylist()[0]
    assert row["mn"] == 2**63 and row["mx"] == 3
    res = engine.aggregate(df, PartitionSpec(by="g"), [ff.min(col("v")).alias("mn"),
                                                       ff.percentile_disc(col("v"), 0.0).alias("p0"),
                                                       ff.percentile_disc(col("v"), 1.0).alias("p1")])
    assert "fb_segmented_quantile" in launches.names()
    row = res.as_arrow().to_pylist()[0]
    assert row == {"g": 0, "mn": 2**63, "p0": 1, "p1": 2**63}


def test_the_nan_at_the_end_of_the_order_reads_as_infinity_on_the_hash_route_only(engine, launches):
    """DESIGN, the f64 MIN / MAX paragraph of K6: an accumulator that never moved reads as +inf / -inf, so MIN over
    only 0x7FFF...F is +inf and MAX over only 0xFFFF...F is -inf on the hash route; the scans (K9) keep the bits."""
    hi, lo = np.array([0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF], np.uint64).view(np.float64)
    t = pa.table({"g": pa.array([0, 0, 1, 1], pa.int64()), "v": pa.array([hi, hi, lo, lo], pa.float64()),
                  "p": pa.array([0, 1, 0, 1], pa.int64())})
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    res = engine.aggregate(df, PartitionSpec(by="g"), [ff.min(col("v")).alias("mn"), ff.max(col("v")).alias("mx")])
    assert "fb_groupby_u64" in launches.names()
    a = res.as_arrow().sort_by("g")
    mn, mx = (R.canonical(a.column(c)) for c in ("mn", "mx"))
    assert [og.bits_of(x) for x in mn] == [og.POS_INF_BITS, og.bits_of(lo)]
    assert [og.bits_of(x) for x in mx] == [og.bits_of(hi), og.NEG_INF_BITS]
    launches.calls.clear()
    w = fa.transform(df, ColumnMap(col("g"), ff.min(col("v")).over().alias("mn"), ff.max(col("v")).over().alias("mx")),
                     schema="g:long,mn:double,mx:double", partition=PartitionSpec(by="g", presort="p asc"),
                     engine=engine, as_fugue=True).as_arrow().sort_by("g")
    assert "fb_segmented_scan" in launches.names()
    assert [og.bits_of(x) for x in R.canonical(w.column("mn"))] == [og.bits_of(hi)] * 2 + [og.bits_of(lo)] * 2
    assert [og.bits_of(x) for x in R.canonical(w.column("mx"))] == [og.bits_of(hi)] * 2 + [og.bits_of(lo)] * 2
