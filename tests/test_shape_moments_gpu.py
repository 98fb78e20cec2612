"""SKEWNESS / SKEWNESS_POP / KURTOSIS / KURTOSIS_POP on the device against the exact reference
(oracle/shape_moments.py).

Tolerances are the rounding bounds of DESIGN §7m, coded in ``oracle.shape_moments.sums_bound`` (the central sums M2,
M3, M4) and ``result_bound`` (a statistic): the hash group-by's corrected sums about its summed mean (``"hash"``) and
the scan's pairwise updates (``"scan"``).  A constant group gives exactly 0 on both routes and a NaN or +-inf gives
NaN.  Where every sum is exact (small integers in groups of 2^k rows) K6's central sums equal the reference exactly.
"""
import math
from fractions import Fraction
from typing import Any, Callable, Dict, List, Optional, Sequence

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import _lib
from fugue_b200 import aggregates as A
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import shape_moments as OS

DEV = torch.device("cuda", 0)
U = OS.U
FUNCS = OS.FUNCS
SHAPE_OPS = [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64, K.AGG_DEV3_F64, K.AGG_DEV4_F64, K.AGG_MIN_F64,
             K.AGG_MAX_F64]
_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


# ---- checks ------------------------------------------------------------------------------------------
def check_sums(m_got: int, got: List[float], vals: List[Optional[float]], route: str) -> None:
    """(m, M2, M3, M4) of a group or a running prefix against the exact central sums."""
    vals = [float(x) for x in vals if x is not None]
    assert m_got == len(vals)
    if not vals:
        return
    m, *ex = OS.central_sums(vals)
    if ex[0] is None:
        assert all(math.isnan(g) for g in got), (vals[:5], got)
        return
    if ex[0] == 0:
        assert got == [0.0, 0.0, 0.0], (vals[:5], got)
        return
    for g, e, b in zip(got, ex, OS.sums_bound(vals, route)):
        assert abs(g - float(e)) <= b, (len(vals), got, [float(q) for q in ex])


def check_result(fn: str, got: Optional[float], vals: List[Optional[float]], route: str) -> None:
    vals = [float(x) for x in vals if x is not None]
    check_finished(fn, got, OS.central_sums(vals), lambda: OS.sums_bound(vals, route))


def check_finished(fn: str, got: Optional[float], mom: OS.Moments, bounds: Callable[[], Sequence[float]]) -> None:
    """``check_result`` from the exact (m, M2, M3, M4) of ``OS.central_sums``; ``bounds()`` gives the bounds on the
    computed M2, M3, M4 and is called only for finite values that are not all equal."""
    want = OS.finish(fn, mom)
    if want is None:
        assert got is None, (fn, mom[0], got)
        return
    assert got is not None, (fn, mom[0])
    if math.isnan(want):
        assert math.isnan(got), (fn, mom[0], got)
        return
    if mom[1] == 0:
        assert got == 0.0, (fn, mom[0], got)
        return
    assert abs(got - want) <= OS.box_bound(fn, mom[0], [float(q) for q in mom[1:]], bounds()), \
        (fn, mom[0], got, want)


# ---- K6 kernel paths ---------------------------------------------------------------------------------
class Launches:
    """(nrows, naggs, num_parts, batched) of every ``fb_groupby_u64`` call."""

    def __init__(self, monkeypatch: Any):
        lib = _lib.load()
        real = lib.fb_groupby_u64
        self.calls: List[tuple] = []

        def spy(*a: Any) -> int:
            self.calls.append((a[2], a[5], a[10], bool(a[13])))
            return real(*a)

        monkeypatch.setattr(lib, "fb_groupby_u64", spy)

    def path(self, nrows: int) -> str:
        _, naggs, parts, batched = [c for c in self.calls if c[0] == nrows][-1]
        if parts == 0:
            return "generic"
        if batched:
            return "batched"
        return f"lean{naggs}" if 1 <= naggs <= 4 else "region"


@pytest.fixture
def launches(monkeypatch):
    return Launches(monkeypatch)


def _groupby(keys, kv, v, vm, ops, partition):
    kt = torch.from_numpy(keys).to(DEV)
    kvt = None if kv is None else torch.from_numpy(kv).to(DEV)
    vt = torch.from_numpy(v).to(DEV)
    mt = None if vm is None else torch.from_numpy(vm).to(DEV)
    vals = [None if o == K.AGG_COUNT else vt for o in ops]
    gk, gv, ga, ng = K.groupby_u64(kt, kvt, vals, [mt] * len(ops), ops, partition=partition)
    gkeys = [(k if ok else None) for k, ok in zip(gk.cpu().tolist(), [1] * ng if gv is None else gv.cpu().tolist())]
    return gkeys, ga


def run_k6(keys, kv, v, vm, partition: bool) -> Dict[Any, tuple]:
    """(m, [M2, M3, M4]) per key through ``groupby_u64`` with the eight accumulators of a shape statistic, the
    central sums formed as the engine forms them."""
    gkeys, ga = _groupby(keys, kv, v, vm, SHAPE_OPS, partition)
    m, *q = A.shape_moments(ga, tuple(range(8)))
    q = [x.cpu().tolist() for x in q]
    return {k: (c, [q[0][i], q[1][i], q[2][i]]) for i, (k, c) in enumerate(zip(gkeys, m.cpu().tolist()))}


def edge_data(n: int, seed: int = 0):
    """Values in random groups (dyadic, N(0, 1) and cubed normals for skew), plus the edge groups: m = 0 .. 4,
    constant, NaN, +-inf, the NULL key and the all-ones key (the table's EMPTY pattern)."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, max(n // 20, 1), n).astype(np.int64)
    v = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0
    normal = rng.random(n) < 0.3
    v[normal] = rng.standard_normal(int(normal.sum())) ** 3
    vm = (rng.random(n) > 0.1).astype(np.uint8)
    kv = (rng.random(n) > 0.02).astype(np.uint8)
    edges = [(10**9 + 0, [None, None, None]), (10**9 + 1, [2.5]), (10**9 + 2, [1.0, 4.0]),
             (10**9 + 3, [1.0, 2.0, 7.0]), (10**9 + 4, [-1.0, 0.5, 3.0, 3.25]), (10**9 + 5, [0.1] * 50),
             (10**9 + 6, [1.0, math.nan, 2.0]), (10**9 + 7, [math.inf, 1.0]), (10**9 + 8, [-math.inf, math.inf]),
             (-1, [7.0, 9.0, 11.5, 20.0])]
    pos = 0
    for key, vals in edges:
        for x in vals:
            keys[pos], kv[pos], vm[pos], v[pos] = key, 1, 0 if x is None else 1, 0.0 if x is None else x
            pos += 1
    return keys, kv, v, vm


def expected_groups(keys, kv, v, vm) -> Dict[Any, List[Optional[float]]]:
    groups: Dict[Any, List[Optional[float]]] = {}
    for k, ok, x, xm in zip(keys.tolist(), kv.tolist(), v.tolist(), vm.tolist()):
        groups.setdefault(k if ok else None, []).append(x if xm else None)
    return groups


@pytest.mark.parametrize("path", ["generic", "region", "batched"])
def test_k6_paths_against_the_oracle(path, launches, monkeypatch):
    n = 60_000
    keys, kv, v, vm = edge_data(n)
    if path == "batched":
        monkeypatch.setattr(K, "GROUPBY_BATCHED", True)
    got = run_k6(keys, kv, v, vm, partition=path != "generic")
    assert launches.path(n) == path
    groups = expected_groups(keys, kv, v, vm)
    assert set(got) == set(groups)
    for k, vals in groups.items():
        check_sums(*got[k], vals, "hash")


def test_k6_lean_layout_adds_the_third_and_fourth_powers(launches):
    """A shape statistic needs eight accumulators, more than the lean kernel takes; SUM, COUNT, DEV3 and DEV4 alone
    run its layout (``fb_groupby_dev_kernel<true, true>``): the sums of d^3 and d^4 about SUM / COUNT."""
    n = 200_000
    rng = np.random.default_rng(1)
    keys = rng.integers(0, 5000, n).astype(np.int64)
    v = rng.standard_normal(n) * 3 + 1
    vm = (rng.random(n) > 0.1).astype(np.uint8)
    gkeys, ga = _groupby(keys, None, v, vm, [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV3_F64, K.AGG_DEV4_F64], True)
    assert launches.path(n) == "lean4"
    s, c = ga[0].view(torch.float64).cpu().tolist(), ga[1].cpu().tolist()
    d3, d4 = (ga[i].view(torch.float64).cpu().tolist() for i in (2, 3))
    groups = expected_groups(keys, np.ones(n, np.uint8), v, vm)
    for i, k in enumerate(gkeys[:400]):
        vals = [x for x in groups[k] if x is not None]
        mean = s[i] / c[i]  # the kernel's own mean, correctly rounded as on the host
        ds = [Fraction(x) - Fraction(mean) for x in vals]
        for got, p in ((d3[i], 3), (d4[i], 4)):
            ex = float(sum(d ** p for d in ds))
            # d, its powers and the atomic sum: at most (m + 6) roundings of sum |d|^p
            assert abs(got - ex) <= (len(vals) + 6) * U * float(sum(abs(d) ** p for d in ds)), (k, p, got, ex)


def test_k6_rejects_a_power_without_its_sum_and_count():
    v = torch.arange(10, dtype=torch.float64, device=DEV)
    k = torch.zeros(10, dtype=torch.int64, device=DEV)
    for ops in ([K.AGG_COUNT, K.AGG_DEV3_F64], [K.AGG_SUM_F64, K.AGG_DEV4_F64]):
        vals = [None if o == K.AGG_COUNT else v for o in ops]
        with pytest.raises(_lib.FugueB200KernelError, match="needs a SUM_F64 and a COUNT"):
            K.groupby_u64(k, None, vals, [None] * len(ops), ops, partition=False)


def test_k6_dyadic_sums_are_exact():
    """Integers in [-8, 8] in groups of 64 rows: the summed mean is exact, every d^k and every sum fits 53 bits,
    so M2, M3 and M4 equal the reference exactly and a statistic is within the finisher's own roundings."""
    rng = np.random.default_rng(4)
    ngroups = 4096
    keys = np.repeat(rng.permutation(ngroups * 7)[:ngroups].astype(np.int64), 64)
    v = rng.integers(-8, 9, len(keys)).astype(np.float64)
    got = run_k6(keys, None, v, None, partition=True)
    groups = expected_groups(keys, np.ones(len(v), np.uint8), v, np.ones(len(v), np.uint8))
    for k, vals in groups.items():
        m, *ex = OS.central_sums(vals)
        assert got[k][0] == m and got[k][1] == [float(q) for q in ex], (k, got[k], ex)
        for fn in FUNCS:
            r, _ = A.shape_of(fn, torch.tensor([m]), *(torch.tensor([q], dtype=torch.float64) for q in got[k][1]))
            want = OS.result(fn, vals)
            scale = abs(want) + (3 * (m - 1) ** 2 / ((m - 2) * (m - 3)) if fn == "KURTOSIS" else 3)
            assert abs(r.item() - want) <= 8 * U * scale


def test_high_mean_and_the_naive_formula_fails_the_same_bound():
    """Mean 1e9, sigma 1e-3: the corrected sums stay within their bound; the textbook power sums do not."""
    rng = np.random.default_rng(9)
    ngroups, per = 200, 500
    keys = np.repeat(np.arange(ngroups, dtype=np.int64), per)
    v = 1e9 + (rng.standard_normal(ngroups * per) + rng.standard_normal(ngroups * per) ** 2) * 1e-3
    res = fa.aggregate(_df(pa.table({"k": keys, "v": v})), "k", engine=_engine(), as_fugue=True,
                       s=f.skewness(col("v")), k2=f.kurtosis(col("v"))).as_arrow().to_pylist()
    groups = expected_groups(keys, np.ones(len(v), np.uint8), v, np.ones(len(v), np.uint8))
    assert len(res) == ngroups
    naive_fails = 0
    for r in res:
        vals = groups[r["k"]]
        for fn, out in (("SKEWNESS", "s"), ("KURTOSIS", "k2")):
            check_result(fn, r[out], vals, "hash")
            naive_fails += abs(OS.naive_power_sums(fn, vals) - OS.result(fn, vals)) > OS.result_bound(fn, vals, "hash")
    assert naive_fails == 2 * ngroups


# ---- engine calls ------------------------------------------------------------------------------------
def _table(rng, n, ngroups=40):
    return pa.table({
        "k": pa.array(rng.integers(0, ngroups, n), mask=rng.random(n) < 0.03),
        "k2": pa.array(rng.integers(0, 3, n).astype(np.int8)),
        "v": pa.array(rng.gamma(2.0, 3.0, n) + 5.0, mask=rng.random(n) < 0.1),
        "i": pa.array(rng.integers(-1000, 1000, n).astype(np.int32)),
    })


def _rows_by(tbl: pa.Table, keys: List[str]):
    out: Dict[Any, List[dict]] = {}
    for r in tbl.to_pylist():
        out.setdefault(tuple(r[k] for k in keys), []).append(r)
    return out


def _check_agg(res: pa.Table, tbl: pa.Table, keys: List[str], spec: Dict[str, tuple], route: str = "hash") -> None:
    """spec: output column -> (head, function of a row giving the argument)."""
    groups = _rows_by(tbl, keys)
    got = res.to_pylist()
    assert len(got) == max(len(groups), 0 if keys else 1)
    for r in got:
        rows = groups.get(tuple(r[k] for k in keys), [])
        for out, (head, arg) in spec.items():
            check_result(head, r[out], [arg(x) for x in rows], route)


ALL = {"a": f.skewness(col("v")), "b": f.skew(col("i")), "c": f.skewness_pop(col("v")), "d": f.kurtosis(col("v")),
       "e": f.kurt(col("i")), "g": f.kurtosis_pop(col("v")), "sd": f.stddev(col("v")), "s": f.sum(col("v"))}
ALL_SPEC = {"a": ("SKEWNESS", lambda r: r["v"]), "b": ("SKEWNESS", lambda r: r["i"]),
            "c": ("SKEWNESS_POP", lambda r: r["v"]), "d": ("KURTOSIS", lambda r: r["v"]),
            "e": ("KURTOSIS", lambda r: r["i"]), "g": ("KURTOSIS_POP", lambda r: r["v"])}


def test_aggregate_all_keyed_and_global():
    tbl = _table(np.random.default_rng(1), 20_000)
    for keys in (["k"], ["k", "k2"], []):
        res = fa.aggregate(_df(tbl), keys or None, engine=_engine(), as_fugue=True, **ALL).as_arrow()
        assert all(res.schema.field(c).type == pa.float64() for c in ALL_SPEC)
        _check_agg(res, tbl, keys, ALL_SPEC)


def test_aggregate_matches_pandas():
    rng = np.random.default_rng(2)
    pdf = pd.DataFrame({"k": rng.integers(0, 300, 30_000), "v": rng.standard_t(4, 30_000) * 10})
    res = fa.aggregate(pdf, "k", s=f.skew(col("v")), t=f.kurt(col("v")), engine=_engine(),
                       as_fugue=True).as_pandas().sort_values("k").reset_index(drop=True)
    want = pdf.groupby("k")["v"]
    assert np.allclose(res["s"], want.skew().to_numpy(), rtol=1e-10, atol=1e-12)
    assert np.allclose(res["t"], want.apply(lambda s: s.kurt()).to_numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("tp", [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(),
                                pa.uint64(), pa.float16(), pa.float32(), pa.float64()])
def test_every_numeric_storage_type(tp):
    rng = np.random.default_rng(3)
    n = 5000
    x = rng.integers(0, 100, n) ** 2 // 100
    tbl = pa.table({"k": rng.integers(0, 30, n), "x": pa.array(x, mask=rng.random(n) < 0.1).cast(tp)})
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, a=f.skewness(col("x")),
                       b=f.kurtosis_pop(col("x"))).as_arrow()
    _check_agg(res, tbl, ["k"], {"a": ("SKEWNESS", lambda r: r["x"]), "b": ("KURTOSIS_POP", lambda r: r["x"])})


def test_empty_table():
    tbl = pa.table({"k": pa.array([], pa.int64()), "v": pa.array([], pa.float64())})
    e = _engine()
    res = fa.aggregate(_df(tbl), None, engine=e, as_fugue=True, a=f.skew(col("v")), s=f.sum(col("v"))).as_arrow()
    assert res.to_pylist() == [{"a": None, "s": None}]
    res = fa.aggregate(_df(tbl), "k", engine=e, as_fugue=True, a=f.kurt(col("v"))).as_arrow()
    assert res.num_rows == 0
    res = fa.aggregate(_df(tbl), None, engine=e, as_fugue=True, a=f.kurtosis_pop(col("v")),
                       m=f.median(col("v"))).as_arrow()
    assert res.to_pylist() == [{"a": None, "m": None}]


def test_median_beside_kurtosis_takes_the_sorted_route():
    tbl = _table(np.random.default_rng(6), 10_000)
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, m=f.median(col("v")),
                       **{o: ALL[o] for o in ALL_SPEC}).as_arrow()
    _check_agg(res, tbl, ["k"], ALL_SPEC, route="scan")
    res = fa.aggregate(_df(tbl), None, engine=_engine(), as_fugue=True, m=f.median(col("v")),
                       **{o: ALL[o] for o in ALL_SPEC}).as_arrow()
    _check_agg(res, tbl, [], ALL_SPEC, route="scan")


def test_three_columns_take_the_sorted_route():
    tbl = _table(np.random.default_rng(7), 10_000)
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, a=f.kurt(col("v")), b=f.skew(col("i")),
                       c=f.kurtosis(col("k2"))).as_arrow()
    _check_agg(res, tbl, ["k"], {"a": ("KURTOSIS", lambda r: r["v"]), "b": ("SKEWNESS", lambda r: r["i"]),
                                 "c": ("KURTOSIS", lambda r: r["k2"])}, route="scan")


def test_select_with_where_having_and_expressions():
    tbl = _table(np.random.default_rng(4), 20_000)
    sk = f.skew(col("v"))
    res = fa.select(_df(tbl), col("k"), sk.alias("s"), f.kurtosis_pop(col("v") * 2 + col("i")).alias("p"),
                    (sk / f.stddev(col("v"))).alias("r"), where=col("i") > -500, having=sk > 1.3, engine=_engine(),
                    as_fugue=True).as_arrow()
    flt = tbl.filter(pa.compute.fill_null(pa.compute.greater(tbl.column("i"), -500), False))
    groups = _rows_by(flt, ["k"])
    kept = 0
    for key, rows in groups.items():
        want = OS.result("SKEWNESS", [r["v"] for r in rows])
        if want is not None and abs(want - 1.3) < 1e-9:
            continue  # too close to the HAVING threshold to decide
        kept += want is not None and want > 1.3
    assert res.num_rows == kept
    for r in res.to_pylist():
        rows = groups[(r["k"],)]
        check_result("SKEWNESS", r["s"], [x["v"] for x in rows], "hash")
        check_result("KURTOSIS_POP", r["p"], [None if x["v"] is None else x["v"] * 2 + x["i"] for x in rows], "hash")


def test_raw_sql_every_name():
    rng = np.random.default_rng(5)
    n = 20_000
    pdf = pd.DataFrame({"key": rng.integers(0, 100, n), "v": rng.gamma(3.0, 2.0, n) - 1})
    got = fa.raw_sql("SELECT key, SKEWNESS(v) AS a, skew(v) AS b, Skewness_Pop(v) AS c, KURTOSIS(v) AS d, "
                     "kurt(v) AS e, KURTOSIS_POP(v) AS g FROM", pdf, "GROUP BY key ORDER BY key", engine=_engine(),
                     as_fugue=True).as_pandas()
    groups = {k: g["v"].tolist() for k, g in pdf.groupby("key")}
    for c, fn in (("a", "SKEWNESS"), ("b", "SKEWNESS"), ("c", "SKEWNESS_POP"), ("d", "KURTOSIS"), ("e", "KURTOSIS"),
                  ("g", "KURTOSIS_POP")):
        for k, x in zip(got["key"].tolist(), got[c].tolist()):
            check_result(fn, x, groups[k], "hash")


def test_rejections():
    tbl = pa.table({"k": [1, 2], "s": ["a", "b"], "b": [True, False], "v": [1.0, 2.0]})
    e = _engine()
    for arg in ("s", "b"):
        with pytest.raises(NotImplementedError):
            fa.aggregate(_df(tbl), "k", engine=e, a=f.skew(col(arg)))
    with pytest.raises(NotImplementedError):
        fa.select(_df(tbl), col("k"), f.kurt(col("v")).alias("s"), f.count_distinct(col("v")).alias("c"), engine=e)


# ---- K9 and window maps ------------------------------------------------------------------------------
def test_segmented_shape_moments_kernel_with_empty_and_long_segments():
    rng = np.random.default_rng(7)
    lengths = [0, 1, 2, 3, 4, 0, 2047, 2048, 2049, 5000, 1, 0, 777, 9000, 64]
    n = sum(lengths)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    v = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0 + 100.0
    v[rng.random(n) < 0.001] = np.inf
    v[off[-2]:] = 0.1  # a constant segment
    vm = (rng.random(n) > 0.1).astype(np.uint8)
    args = (torch.from_numpy(off).to(DEV), n, [(torch.from_numpy(v).to(DEV), torch.from_numpy(vm).to(DEV))])
    (cnt, *ms), = K.segmented_shape_moments(*args)
    cnt, ms = cnt.cpu().tolist(), [x.cpu().tolist() for x in ms]
    for a, b in zip(off[:-1], off[1:]):
        vals = [x if ok else None for x, ok in zip(v[a:b].tolist(), vm[a:b].tolist())]
        m = 0
        for i in range(b - a):
            m += vals[i] is not None
            assert cnt[a + i] == m
            if m == 0:
                assert [q[a + i] for q in ms] == [0.0, 0.0, 0.0]
            elif i % 499 == 0 or i == b - a - 1:
                check_sums(cnt[a + i], [q[a + i] for q in ms], vals[:i + 1], "scan")
    # identical bits from run to run (fixed combination order)
    (c2, *ms2), = K.segmented_shape_moments(*args)
    assert c2.cpu().tolist() == cnt
    for x, y in zip(ms, ms2):
        assert np.array_equal(np.asarray(x).view(np.int64), y.cpu().numpy().view(np.int64))


def _window(tbl: pa.Table, cols, by=("k",), presort="t"):
    spec = PartitionSpec(by=list(by), presort=presort)
    schema = "rid:long," + ",".join(f"{c.output_name}:double" for c in cols)
    return fa.transform(_df(tbl), ColumnMap("rid", *cols), schema=schema, partition=spec, engine=_engine(),
                        as_fugue=True).as_arrow()


def test_window_whole_partition_and_running():
    rng = np.random.default_rng(8)
    n = 30_000
    k = rng.integers(0, 6, n)  # partitions longer than a tile (2048 rows)
    k[:1] = 100                # a one-row partition
    k[1:4] = 101               # a partition of NULL values only
    k[4:9] = 102               # a constant partition
    v = rng.gamma(2.0, 5.0, n) + 20.0
    v[4:9] = 3.5
    mask = rng.random(n) < 0.1
    mask[1:4] = True
    mask[4:9] = False
    tbl = pa.table({"rid": np.arange(n), "k": k, "t": rng.permutation(n), "v": pa.array(v, mask=mask)})
    cols = [f.skewness(col("v")).over().alias("sw"), f.kurtosis_pop(col("v")).over().alias("kw"),
            f.skew(col("v")).over(running=True).alias("sr"), f.kurt(col("v")).over(running=True).alias("kr"),
            f.skewness_pop(col("v")).over(running=True).alias("pr"), f.stddev(col("v")).over().alias("sd")]
    out = _window(tbl, cols)
    rows = {r["rid"]: r for r in tbl.to_pylist()}
    res = {r["rid"]: r for r in out.to_pylist()}
    parts: Dict[int, List[dict]] = {}
    for r in sorted(rows.values(), key=lambda r: r["t"]):
        parts.setdefault(r["k"], []).append(r)
    for key, prs in parts.items():
        allv = [r["v"] for r in prs]
        for i, r in enumerate(prs):
            got = res[r["rid"]]
            if i % 701 == 0 or i == len(prs) - 1 or len(prs) < 10:
                check_result("SKEWNESS", got["sw"], allv, "scan")
                check_result("KURTOSIS_POP", got["kw"], allv, "scan")
                check_result("SKEWNESS", got["sr"], allv[:i + 1], "scan")
                check_result("KURTOSIS", got["kr"], allv[:i + 1], "scan")
                check_result("SKEWNESS_POP", got["pr"], allv[:i + 1], "scan")
    again = _window(tbl, cols)
    for c in ("sw", "kw", "sr", "kr", "pr"):
        assert np.array_equal(np.asarray(out.column(c).to_numpy(zero_copy_only=False)).view(np.int64),
                              np.asarray(again.column(c).to_numpy(zero_copy_only=False)).view(np.int64))
