"""VAR_SAMP / VAR_POP / STDDEV_SAMP / STDDEV_POP on the device against the exact reference (oracle/moments.py).

Tolerances are the rounding bounds of the two algorithms (u = 2^-53, kappa = ||x||_2 / sqrt(M2), m values):
  * K6, the corrected two-pass of the hash group-by: |M2 - exact| <= 2 ((m + 2) u M2 + (m u)^2 ||x||^2), i.e. a
    relative error of m u + (m u kappa)^2 (Chan, Golub & LeVeque 1983; the atomic sum of the mean adds at most
    m u sum |x| / m to the shift, whose square enters only through the correction term);
  * K9, the updating moments scan: |M2 - exact| <= 4 m u kappa M2 = 4 m u ||x|| sqrt(M2).
A variance adds one rounding of the quotient, a standard deviation is checked through its square.
"""
import math
from fractions import Fraction
from typing import Any, Dict, List, Optional

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import _lib
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import moments as OM

DEV = torch.device("cuda", 0)
U = 2.0 ** -53
_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


# ---- bounds ------------------------------------------------------------------------------------------
def m2_tol(vals: List[float], scan: bool) -> float:
    m = len(vals)
    ex = float(OM.exact_m2(vals))
    sx2 = float(sum(Fraction(x) ** 2 for x in vals))
    return 4 * m * U * math.sqrt(sx2 * ex) if scan else 2 * ((m + 2) * U * ex + (m * U) ** 2 * sx2)


def check_m2(m_got: int, m2_got: float, vals: List[Optional[float]], scan: bool = False) -> None:
    vals = [float(x) for x in vals if x is not None]
    assert m_got == len(vals)
    if not vals:
        return
    if not all(math.isfinite(x) for x in vals):
        assert math.isnan(m2_got), (vals[:5], m2_got)
        return
    ex = float(OM.exact_m2(vals))
    assert m2_got >= 0 and abs(m2_got - ex) <= m2_tol(vals, scan), (len(vals), m2_got, ex)


def check_result(fn: str, got: Optional[float], vals: List[Optional[float]], scan: bool = False) -> None:
    vals = [float(x) for x in vals if x is not None]
    want = OM.result_exact(fn, vals)
    if want is None:
        assert got is None, (fn, vals, got)
        return
    assert got is not None, (fn, vals)
    if math.isnan(want):
        assert math.isnan(got)
        return
    check_finite_result(fn, got, len(vals), OM.exact_m2(vals), m2_tol(vals, scan))


def check_finite_result(fn: str, got: float, m: int, m2: Fraction, m2_bound: float) -> None:
    """``check_result`` of m finite values (at least the function's minimum count) from their exact M2 and the
    bound on the computed M2."""
    div = m - 1 if fn.endswith("_SAMP") else m
    var = float(m2 / div)
    tol = m2_bound / div + 2 * U * var
    g = got * got if fn.startswith("STDDEV") else got
    assert abs(g - var) <= tol + (4 * U * var if fn.startswith("STDDEV") else 0), (fn, m, got, var)


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


def run_k6(keys: np.ndarray, kv: Optional[np.ndarray], v: np.ndarray, vm: Optional[np.ndarray], partition: bool,
           extra: bool = False) -> Dict[Any, tuple]:
    """(m, M2) per key through ``groupby_u64`` with SUM, COUNT, DEV, DEV2 (and a fifth accumulator with
    ``extra``), M2 formed as the engine does."""
    kt = torch.from_numpy(keys).to(DEV)
    kvt = None if kv is None else torch.from_numpy(kv).to(DEV)
    vt = torch.from_numpy(v).to(DEV)
    mt = None if vm is None else torch.from_numpy(vm).to(DEV)
    vals, vv, ops = [vt, None, vt, vt], [mt] * 4, [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64]
    if extra:
        vals, vv, ops = vals + [vt], vv + [mt], ops + [K.AGG_MAX_F64]
    gk, gv, ga, ng = K.groupby_u64(kt, kvt, vals, vv, ops, partition=partition)
    m = ga[1]
    d = ga[2].view(torch.float64)
    m2 = torch.clamp_min(ga[3].view(torch.float64) - d * d / m.to(torch.float64), 0.0)
    keys_ = gk.cpu().tolist()
    valid = [1] * ng if gv is None else gv.cpu().tolist()
    return {(k if ok else None): (c, q) for k, ok, c, q in zip(keys_, valid, m.cpu().tolist(), m2.cpu().tolist())}


def edge_data(n: int, seed: int = 0):
    """Dyadic values k / 1024 in random groups, plus the edge groups: m = 0, 1, 2, constant, NaN, +-inf, the
    NULL key and the all-ones key (the table's EMPTY pattern), and some N(0, 1) values."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, max(n // 20, 1), n).astype(np.int64)
    v = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0
    normal = rng.random(n) < 0.2
    v[normal] = rng.standard_normal(int(normal.sum()))
    vm = (rng.random(n) > 0.1).astype(np.uint8)
    kv = (rng.random(n) > 0.02).astype(np.uint8)
    edges = [(10**9 + 0, [None, None, None]), (10**9 + 1, [2.5]), (10**9 + 2, [1.0, 4.0]),
             (10**9 + 3, [3.25] * 50), (10**9 + 4, [1.0, math.nan, 2.0]), (10**9 + 5, [math.inf, 1.0]),
             (10**9 + 6, [-math.inf, math.inf]), (-1, [7.0, 9.0, 11.5])]
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


def check_groups(got, groups) -> None:
    assert set(got) == set(groups)
    for k, vals in groups.items():
        check_m2(*got[k], vals)


@pytest.mark.parametrize("path", ["generic", "lean4", "region", "batched"])
def test_k6_paths_against_the_oracle(path, launches, monkeypatch):
    n = 60_000
    keys, kv, v, vm = edge_data(n)
    if path == "batched":
        monkeypatch.setattr(K, "GROUPBY_BATCHED", True)
    got = run_k6(keys, kv, v, vm, partition=path != "generic", extra=path in ("region", "batched"))
    assert launches.path(n) == path
    check_groups(got, expected_groups(keys, kv, v, vm))


def test_k6_one_region_retry(launches):
    """Every key in one hash partition: region mode overflows, and the retry over one region must find the same
    slots in pass B."""
    n = 200_000
    cand = torch.arange(1 << 23, dtype=torch.int64, device=DEV)
    pool = cand[K.partition_ids([cand], K.GROUPBY_PARTITIONS) == 3][:20_000].cpu().numpy()
    rng = np.random.default_rng(3)
    keys = rng.choice(pool, n)
    v = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0
    got = run_k6(keys, None, v, None, partition=True)
    calls = [c for c in launches.calls if c[0] == n]
    assert calls[0][2] == K.GROUPBY_PARTITIONS and calls[-1][2] == 0
    check_groups(got, expected_groups(keys, np.ones(n, np.uint8), v, np.ones(n, np.uint8)))


def test_k6_rejects_a_deviation_without_its_sum_and_count():
    v = torch.arange(10, dtype=torch.float64, device=DEV)
    k = torch.zeros(10, dtype=torch.int64, device=DEV)
    for ops in ([K.AGG_COUNT, K.AGG_DEV_F64], [K.AGG_SUM_F64, K.AGG_DEV2_F64]):
        vals = [None if o == K.AGG_COUNT else v for o in ops]
        with pytest.raises(_lib.FugueB200KernelError, match="needs a SUM_F64 and a COUNT"):
            K.groupby_u64(k, None, vals, [None] * len(ops), ops, partition=False)
    other = v.clone()
    with pytest.raises(_lib.FugueB200KernelError, match="needs a SUM_F64 and a COUNT"):
        K.groupby_u64(k, None, [other, None, v], [None] * 3, [K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64],
                      partition=False)


def test_large_offset_and_the_naive_formula_fails_the_same_bound():
    """Mean 1e9, sigma 1e-3: the corrected two-pass stays within its bound; sum(x^2) - sum(x)^2 / m does not."""
    rng = np.random.default_rng(9)
    ngroups, per = 200, 500
    keys = np.repeat(np.arange(ngroups, dtype=np.int64), per)
    v = 1e9 + rng.standard_normal(ngroups * per) * 1e-3
    got = run_k6(keys, None, v, None, partition=False)
    groups = expected_groups(keys, np.ones(len(v), np.uint8), v, np.ones(len(v), np.uint8))
    check_groups(got, groups)
    naive_fails = 0
    for k, vals in groups.items():
        x = np.asarray(vals)
        naive = float(np.sum(x * x) - np.sum(x) ** 2 / len(x))
        naive_fails += abs(naive - float(OM.exact_m2(vals))) > m2_tol(vals, False)
    assert naive_fails == ngroups


def test_k6_dyadic_million_rows():
    """4 M rows, 65 536 keys, on the partitioned (lean) path: exact integer sums of the reference."""
    rng = np.random.default_rng(4)
    n = 4_000_000
    keys = rng.integers(0, 65_536, n).astype(np.int64)
    k = rng.integers(-(1 << 20) + 1, 1 << 20, n)
    vm = (rng.random(n) > 0.05).astype(np.uint8)
    got = run_k6(keys, None, k / 1024.0, vm, partition=True)
    want = OM.dyadic_group_moments(keys, k, vm)
    for g, (m, ex) in want.items():
        c, q = got[g]
        assert c == m
        # ||x||^2 <= m 2^40 / 2^20: the bound of the module docstring
        assert abs(q - ex) <= 2 * ((m + 2) * U * ex + (m * U) ** 2 * m * 2.0 ** 20), (g, q, ex)


# ---- engine calls ------------------------------------------------------------------------------------
def _table(rng, n, ngroups=40):
    v = rng.normal(5.0, 3.0, n)
    return pa.table({
        "k": pa.array(rng.integers(0, ngroups, n), mask=rng.random(n) < 0.03),
        "k2": pa.array(rng.integers(0, 3, n).astype(np.int8)),
        "v": pa.array(v, mask=rng.random(n) < 0.1),
        "i": pa.array(rng.integers(-1000, 1000, n).astype(np.int32)),
    })


def _rows_by(tbl: pa.Table, keys: List[str]):
    out: Dict[Any, List[dict]] = {}
    for r in tbl.to_pylist():
        out.setdefault(tuple(r[k] for k in keys), []).append(r)
    return out


def _check_agg(res: pa.Table, tbl: pa.Table, keys: List[str], spec: Dict[str, tuple]) -> None:
    """spec: output column -> (head, function of a row giving the argument)."""
    groups = _rows_by(tbl, keys)
    got = res.to_pylist()
    assert len(got) == max(len(groups), 0 if keys else 1)
    for r in got:
        rows = groups.get(tuple(r[k] for k in keys), [])
        for out, (head, arg) in spec.items():
            check_result(head, r[out], [arg(x) for x in rows])


def test_aggregate_all_six_keyed_and_global():
    tbl = _table(np.random.default_rng(1), 20_000)
    e = _engine()
    aggs = {"a": f.var_samp(col("v")), "b": f.variance(col("v")), "c": f.var_pop(col("v")),
            "d": f.stddev_samp(col("v")), "e": f.stddev(col("i")), "g": f.stddev_pop(col("v")),
            "s": f.sum(col("v"))}
    spec = {"a": ("VAR_SAMP", lambda r: r["v"]), "b": ("VAR_SAMP", lambda r: r["v"]),
            "c": ("VAR_POP", lambda r: r["v"]), "d": ("STDDEV_SAMP", lambda r: r["v"]),
            "e": ("STDDEV_SAMP", lambda r: r["i"]), "g": ("STDDEV_POP", lambda r: r["v"])}
    for keys in (["k"], ["k", "k2"], []):
        res = fa.aggregate(_df(tbl), keys or None, engine=e, as_fugue=True, **aggs).as_arrow()
        assert all(res.schema.field(c).type == pa.float64() for c in spec)
        _check_agg(res, tbl, keys, spec)


def test_aggregate_matches_pandas_std():
    rng = np.random.default_rng(2)
    pdf = pd.DataFrame({"k": rng.integers(0, 300, 30_000), "v": rng.normal(0, 10, 30_000)})
    res = fa.aggregate(pdf, "k", s=f.stddev(col("v")), p=f.stddev_pop(col("v")), engine=_engine(),
                       as_fugue=True).as_pandas()
    res = res.sort_values("k").reset_index(drop=True)
    want = pdf.groupby("k")["v"]
    assert np.allclose(res["s"], want.std().to_numpy(), rtol=1e-12, atol=0)
    assert np.allclose(res["p"], want.std(ddof=0).to_numpy(), rtol=1e-12, atol=0)


@pytest.mark.parametrize("tp", [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(),
                                pa.uint64(), pa.float16(), pa.float32(), pa.float64()])
def test_every_numeric_storage_type(tp):
    rng = np.random.default_rng(3)
    n = 5000
    x = rng.integers(0, 100, n)
    tbl = pa.table({"k": rng.integers(0, 30, n), "x": pa.array(x, mask=rng.random(n) < 0.1).cast(tp)})
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, a=f.var_samp(col("x")),
                       b=f.stddev_pop(col("x"))).as_arrow()
    _check_agg(res, tbl, ["k"], {"a": ("VAR_SAMP", lambda r: r["x"]), "b": ("STDDEV_POP", lambda r: r["x"])})


def test_empty_table():
    tbl = pa.table({"k": pa.array([], pa.int64()), "v": pa.array([], pa.float64())})
    e = _engine()
    res = fa.aggregate(_df(tbl), None, engine=e, as_fugue=True, a=f.stddev(col("v")), s=f.sum(col("v"))).as_arrow()
    assert res.to_pylist() == [{"a": None, "s": None}]
    res = fa.aggregate(_df(tbl), "k", engine=e, as_fugue=True, a=f.var_pop(col("v"))).as_arrow()
    assert res.num_rows == 0
    res = fa.aggregate(_df(tbl), None, engine=e, as_fugue=True, a=f.stddev(col("v")), m=f.median(col("v"))).as_arrow()
    assert res.to_pylist() == [{"a": None, "m": None}]


def test_select_with_where_having_and_expressions():
    tbl = _table(np.random.default_rng(4), 20_000)
    e = _engine()
    sd = f.stddev(col("v"))
    res = fa.select(_df(tbl), col("k"), sd.alias("s"), f.var_pop(col("v") * 2 + col("i")).alias("p"),
                    (sd / f.avg(col("v"))).alias("cv"), where=col("i") > -500, having=sd > 2.9, engine=e,
                    as_fugue=True).as_arrow()
    flt = tbl.filter(pa.compute.fill_null(pa.compute.greater(tbl.column("i"), -500), False))
    groups = _rows_by(flt, ["k"])
    kept = 0
    for key, rows in groups.items():
        vals = [r["v"] for r in rows]
        want = OM.result_exact("STDDEV_SAMP", vals)
        if want is not None and not math.isnan(want) and abs(want - 2.9) < 1e-9:
            continue  # too close to the HAVING threshold to decide
        kept += want is not None and want > 2.9
    assert res.num_rows == kept
    for r in res.to_pylist():
        rows = groups[(r["k"],)]
        check_result("STDDEV_SAMP", r["s"], [x["v"] for x in rows])
        check_result("VAR_POP", r["p"], [None if x["v"] is None else x["v"] * 2 + x["i"] for x in rows])
    res = fa.select(_df(tbl), f.variance(col("v")).alias("g"), where=col("k") < 10, engine=e, as_fugue=True).as_arrow()
    flt = tbl.filter(pa.compute.fill_null(pa.compute.less(tbl.column("k"), 10), False))
    check_result("VAR_SAMP", res.column("g")[0].as_py(), flt.column("v").to_pylist())


def test_raw_sql_all_six_names():
    rng = np.random.default_rng(5)
    n = 20_000
    pdf = pd.DataFrame({"key": rng.integers(0, 100, n), "v": rng.standard_normal(n) * 4 + 1})
    got = fa.raw_sql("SELECT key, VAR_SAMP(v) AS a, variance(v) AS b, Var_Pop(v) AS c, STDDEV_SAMP(v) AS d, "
                     "stddev(v) AS e, STDDEV_POP(v) AS g FROM", pdf, "GROUP BY key ORDER BY key", engine=_engine(),
                     as_fugue=True).as_pandas()
    want = pdf.groupby("key")["v"]
    for c, w in (("a", want.var()), ("b", want.var()), ("c", want.var(ddof=0)), ("d", want.std()),
                 ("e", want.std()), ("g", want.std(ddof=0))):
        assert np.allclose(got[c].to_numpy(), w.to_numpy(), rtol=1e-12, atol=0), c


def test_median_beside_stddev_takes_the_sorted_route():
    tbl = _table(np.random.default_rng(6), 10_000)
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, m=f.median(col("v")), s=f.stddev(col("v")),
                       p=f.var_pop(col("i"))).as_arrow()
    _check_agg(res, tbl, ["k"], {"s": ("STDDEV_SAMP", lambda r: r["v"]), "p": ("VAR_POP", lambda r: r["i"])})


def test_rejections():
    tbl = pa.table({"k": [1, 2], "s": ["a", "b"], "b": [True, False], "v": [1.0, 2.0]})
    e = _engine()
    for arg in ("s", "b"):
        with pytest.raises(NotImplementedError):
            fa.aggregate(_df(tbl), "k", engine=e, a=f.stddev(col(arg)))
    with pytest.raises(NotImplementedError):
        fa.select(_df(tbl), col("k"), f.stddev(col("v")).alias("s"), f.count_distinct(col("v")).alias("c"), engine=e)


# ---- window maps -------------------------------------------------------------------------------------
def test_segmented_moments_kernel_with_empty_and_long_segments():
    rng = np.random.default_rng(7)
    lengths = [0, 1, 2, 3, 0, 2047, 2048, 2049, 5000, 1, 0, 777, 9000]
    n = sum(lengths)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    v = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0 + 1e6
    v[rng.random(n) < 0.001] = np.inf
    vm = (rng.random(n) > 0.1).astype(np.uint8)
    (cnt, m2), = K.segmented_moments(torch.from_numpy(off).to(DEV), n,
                                     [(torch.from_numpy(v).to(DEV), torch.from_numpy(vm).to(DEV))])
    cnt, m2 = cnt.cpu().tolist(), m2.cpu().tolist()
    for a, b in zip(off[:-1], off[1:]):
        run = OM.running_moments([x if ok else None for x, ok in zip(v[a:b].tolist(), vm[a:b].tolist())])
        for i, (m, _) in enumerate(run):
            vals = [x for x, ok in zip(v[a:a + i + 1].tolist(), vm[a:a + i + 1].tolist()) if ok] if i % 499 == 0 \
                or i == b - a - 1 else None
            assert cnt[a + i] == m
            if vals is not None:
                check_m2(cnt[a + i], m2[a + i], vals, scan=True)
            elif m == 0:
                assert m2[a + i] == 0.0


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
    v = rng.normal(50.0, 5.0, n)
    mask = rng.random(n) < 0.1
    mask[1:4] = True
    tbl = pa.table({"rid": np.arange(n), "k": k, "t": rng.permutation(n), "v": pa.array(v, mask=mask)})
    cols = [f.stddev(col("v")).over().alias("sw"), f.var_pop(col("v")).over().alias("pw"),
            f.variance(col("v")).over(running=True).alias("vr"), f.stddev_pop(col("v")).over(running=True).alias("sr")]
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
            if i % 701 == 0 or i == len(prs) - 1:
                check_result("STDDEV_SAMP", got["sw"], allv, scan=True)
                check_result("VAR_POP", got["pw"], allv, scan=True)
                check_result("VAR_SAMP", got["vr"], allv[:i + 1], scan=True)
                check_result("STDDEV_POP", got["sr"], allv[:i + 1], scan=True)
    # identical bits from run to run (fixed combination order)
    again = _window(tbl, cols)
    for c in ("sw", "pw", "vr", "sr"):
        assert np.array_equal(np.asarray(out.column(c).to_numpy(zero_copy_only=False)).view(np.int64),
                              np.asarray(again.column(c).to_numpy(zero_copy_only=False)).view(np.int64))
