"""CORR, COVAR_POP / COVAR_SAMP and the REGR_* aggregates on the device against the exact reference
(oracle/comoments.py).

Tolerances are the rounding bounds of the two algorithms, with u = 2^-53, m pair rows, ||x|| = sqrt(sum x^2) over
them and Sxx, Syy, Sxy the exact sums:
  * K6, the corrected two-pass of the hash group-by.  The atomic sums of x and y give means off by dx, dy with
    |dx| <= m u ||x|| / sqrt(m).  Pass B sums (x - mean x - dx)(y - mean y - dy) = Sxy + m dx dy exactly, and the
    correction DEVx DEVy / m removes m dx dy, so what is left is the rounding of the m products and of their
    atomic sum (at most (m + 2) u of sum |x - mean x| |y - mean y| <= (m + 2) u sqrt(Sxx Syy) by Cauchy-Schwarz)
    and the second-order term of the shifts:
        |Sxy^ - Sxy| <= 2 ((m + 2) u sqrt(Sxx Syy) + (m u)^2 ||x|| ||y||)
    and, as in DESIGN §7i, |Sxx^ - Sxx| <= 2 ((m + 2) u Sxx + (m u)^2 ||x||^2), Syy alike.  A mean is SUM / COUNT:
    |mean^ - mean| <= (m + 1) u max |x|.
  * K9, the co-moments scan.  Every combine adds dx dy na nb / n with dx, dy the differences of two means that
    are each within a few u of the exact means of their runs; summed over the combination tree:
        |Sxy^ - Sxy| <= 4 m u max(||x|| sqrt(Syy), ||y|| sqrt(Sxx))
    and |Sxx^ - Sxx| <= 4 m u ||x|| sqrt(Sxx) as for the moments scan (§7i).  An updated mean is a convex
    combination of two means with at most 4 u max |x| of new error per level: |mean^ - mean| <= 4 m u max |x|.
A result is checked against the range its formula takes over the box [S - e, S + e] of those bounds (corners, and
Sxy = 0 when the box holds it), widened by the rounding of the formula itself (4 u of its magnitude).  The NULL
rules are checked exactly: the constant-column rule makes Sxx exactly 0 on both routes when x is constant.
"""
import itertools
import math
from fractions import Fraction
from typing import Any, Dict, List, Optional, Sequence, Tuple

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
from fugue_b200.column import BIVARIATES, col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.execution_engine import B200ExecutionEngine
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import comoments as OC

DEV = torch.device("cuda", 0)
U = 2.0 ** -53
FUNCS = sorted(BIVARIATES)
_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


def build(fn: str, x: Any, y: Any):
    """``fn`` of the pair (x, y), in SQL's argument order."""
    b = getattr(f, fn.lower())
    return b(y, x) if fn.startswith("REGR_") else b(x, y)


# ---- bounds ------------------------------------------------------------------------------------------
def errors(pairs: Sequence[Tuple[float, float]], scan: bool) -> Tuple[OC.State, Tuple[float, ...]]:
    st = OC.exact_state(pairs)
    m = len(pairs)
    if m == 0 or isinstance(st[3], float):
        return st, (0.0,) * 5
    sxx, syy = float(st[3]), float(st[4])
    nx = math.sqrt(sum(x * x for x, _ in pairs))
    ny = math.sqrt(sum(y * y for _, y in pairs))
    ax, ay = max(abs(x) for x, _ in pairs), max(abs(y) for _, y in pairs)
    if scan:
        e = (4 * m * U * ax, 4 * m * U * ay, 4 * m * U * nx * math.sqrt(sxx), 4 * m * U * ny * math.sqrt(syy),
             4 * m * U * max(nx * math.sqrt(syy), ny * math.sqrt(sxx)))
    else:
        e = ((m + 1) * U * ax, (m + 1) * U * ay, 2 * ((m + 2) * U * sxx + (m * U) ** 2 * nx * nx),
             2 * ((m + 2) * U * syy + (m * U) ** 2 * ny * ny),
             2 * ((m + 2) * U * math.sqrt(sxx * syy) + (m * U) ** 2 * nx * ny))
    return st, e


def formula(fn: str, m: int, mx: float, my: float, sxx: float, syy: float, sxy: float) -> float:
    if fn == "COVAR_POP":
        return sxy / m
    if fn == "COVAR_SAMP":
        return sxy / (m - 1)
    if fn in ("REGR_AVGX", "REGR_AVGY", "REGR_SXX", "REGR_SYY", "REGR_SXY"):
        return {"REGR_AVGX": mx, "REGR_AVGY": my, "REGR_SXX": sxx, "REGR_SYY": syy, "REGR_SXY": sxy}[fn]
    if fn == "REGR_SLOPE":
        return sxy / sxx
    if fn == "REGR_INTERCEPT":
        return my - sxy / sxx * mx
    if fn == "REGR_R2":
        return 1.0 if syy == 0 else min(1.0, max(0.0, sxy * sxy / (sxx * syy)))
    return min(1.0, max(-1.0, sxy / (math.sqrt(sxx) * math.sqrt(syy))))  # CORR


def check(fn: str, got: Optional[float], pairs: Sequence[Tuple[float, float]], scan: bool,
          pre: Optional[Tuple] = None) -> None:
    """``pre``: ``errors(pairs, scan)`` when the caller checks several functions of the same rows."""
    st, e = pre if pre is not None else errors(pairs, scan)
    want = OC.result_of_state(fn, st)
    if want is None:
        assert got is None, (fn, len(pairs), got)
        return
    assert got is not None, (fn, len(pairs), want)
    if fn == "REGR_COUNT":
        assert got == want
        return
    if math.isnan(want) or math.isinf(want):
        assert got == want or (math.isnan(want) and math.isnan(got)), (fn, got, want)
        return
    m = st[0]
    centre = [float(v) for v in st[1:]]
    axes = []
    for i, (c, d) in enumerate(zip(centre, e)):
        pts = [c - d, c + d]
        if i in (2, 3):
            pts = [max(p, 0.0) for p in pts]
        if i == 4 and c - d <= 0 <= c + d:
            pts.append(0.0)
        axes.append(pts)
    vals = []
    for mx, my, sxx, syy, sxy in itertools.product(*axes):
        if (sxx == 0 and fn in ("REGR_SLOPE", "REGR_INTERCEPT", "REGR_R2", "CORR")) or (syy == 0 and fn == "CORR"):
            return  # the bound does not keep the denominator off 0: nothing to check beyond the NULL rule
        vals.append(formula(fn, m, mx, my, sxx, syy, sxy))
    lo, hi = min(vals), max(vals)
    slack = 4 * U * max(abs(lo), abs(hi))
    if fn == "REGR_INTERCEPT":
        slack += 4 * U * (abs(centre[1]) + abs(float(st[5] / st[3]) * centre[0]))
    assert lo - slack <= got <= hi + slack, (fn, m, got, want, lo, hi)


def check_row(row: Dict[str, Any], names: Dict[str, str], pairs, scan: bool) -> None:
    """names: output column -> function."""
    pre = errors(pairs, scan)
    for out, fn in names.items():
        check(fn, row[out], pairs, scan, pre)


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


def run_k6(keys: np.ndarray, x: np.ndarray, xm: Optional[np.ndarray], y: np.ndarray, ym: Optional[np.ndarray],
           partition: bool) -> Dict[Any, Tuple]:
    """(m, mean x, mean y, Sxx, Syy, Sxy) per key through ``groupby_u64`` with the engine's 12 pair accumulators."""
    tbl = pa.table({"x": pa.array(x, mask=None if xm is None else xm == 0),
                    "y": pa.array(y, mask=None if ym is None else ym == 0)})
    t = B200Table.from_arrow(tbl, DEV)
    vals, vv, ops = [], [], []

    def add(v, m, op):
        vals.append(v)
        vv.append(m)
        ops.append(op)
        return len(ops) - 1

    slots = B200ExecutionEngine._pair_accumulators(t, f.corr("x", "y"), ("x", "y"), add, {}, {})
    assert len(ops) == 12 and len({id(m) for m in vv}) == 1  # one pair validity tensor
    gk, _, ga, ng = K.groupby_u64(torch.from_numpy(keys).to(DEV), None, vals, vv, ops, partition=partition)
    st = [s.cpu().tolist() for s in B200ExecutionEngine._pair_moments(ga, slots)]
    return {k: tuple(s[i] for s in st) for i, k in enumerate(gk.cpu().tolist())}


def edge_data(n: int, seed: int = 0):
    """Dyadic x and correlated y in random groups, plus the edge groups of the hash path."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, max(n // 30, 1), n).astype(np.int64)
    x = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0
    y = 0.5 * x + rng.integers(-(1 << 18), 1 << 18, n) / 1024.0
    xm = (rng.random(n) > 0.08).astype(np.uint8)
    ym = (rng.random(n) > 0.08).astype(np.uint8)
    N = None
    edges = [(10**9, [(0.1, 2.0), (0.1, 3.0), (0.1, -1.0)] * 7),            # constant x = 0.1: Sxx = Sxy = +0
             (10**9 + 1, [(2.5, 1.0)]),                                     # one pair row
             (10**9 + 2, [(N, 1.0), (1.0, 2.0), (3.0, 5.0), (4.0, N)]),     # NULLs in x only and in y only
             (10**9 + 3, [(N, N), (N, 2.0), (1.0, N)]),                     # no pair row at all
             (10**9 + 4, [(1.0, 2.0), (math.nan, 1.0), (2.0, 3.0)]),        # NaN in x
             (10**9 + 5, [(1.0, math.inf), (2.0, 1.0), (3.0, 0.0)]),        # +inf in y
             (10**9 + 6, [(-math.inf, 1.0), (math.inf, 2.0)]),              # both infinities
             (10**9 + 7, [(1.0, 0.1), (2.0, 0.1), (7.0, 0.1)]),             # constant y: CORR NULL, R2 = 1
             (10**9 + 8, [(N, 1.0), (N, 2.0)])]                             # all x NULL
    pos = 0
    for key, rows in edges:
        for a, b in rows:
            keys[pos] = key
            xm[pos], ym[pos] = a is not None, b is not None
            x[pos], y[pos] = (0.0 if a is None else a), (0.0 if b is None else b)
            pos += 1
    return keys, x, xm, y, ym


def expected(keys, x, xm, y, ym) -> Dict[Any, List[Tuple[float, float]]]:
    out: Dict[Any, List[Tuple[float, float]]] = {}
    for k, a, am, b, bm in zip(keys.tolist(), x.tolist(), xm.tolist(), y.tolist(), ym.tolist()):
        out.setdefault(k, [])
        if am and bm:
            out[k].append((a, b))
    return out


def check_states(got: Dict[Any, Tuple], want: Dict[Any, List], scan: bool = False) -> None:
    from fugue_b200.colmap import bivariate_of

    assert set(got) == set(want)
    for k, pairs in want.items():
        m, mx, my, sxx, syy, sxy = got[k]
        assert m == len(pairs)
        t = [torch.tensor([m])] + [torch.tensor([v], dtype=torch.float64) for v in (mx, my, sxx, syy, sxy)]
        pre = errors(pairs, scan)
        for fn in FUNCS:
            v, ok = bivariate_of(fn, *t)
            check(fn, v.item() if ok is None or ok.item() else None, pairs, scan, pre)


@pytest.mark.parametrize("path", ["generic", "region", "batched"])
def test_k6_paths_against_the_oracle(path, launches, monkeypatch):
    n = 60_000
    keys, x, xm, y, ym = edge_data(n)
    if path == "batched":
        monkeypatch.setattr(K, "GROUPBY_BATCHED", True)
    got = run_k6(keys, x, xm, y, ym, partition=path != "generic")
    assert launches.path(n) == path  # 12 accumulators never take the lean kernel
    check_states(got, expected(keys, x, xm, y, ym))
    const = got[10**9]
    assert const[3] == 0.0 and const[5] == 0.0 and not math.copysign(1.0, const[5]) < 0  # Sxx, Sxy exactly +0


def test_k6_one_region_retry(launches):
    """Every key in one hash partition: region mode overflows, and the retry over one region must find the same
    slots in pass B."""
    n = 200_000
    cand = torch.arange(1 << 23, dtype=torch.int64, device=DEV)
    pool = cand[K.partition_ids([cand], K.GROUPBY_PARTITIONS) == 3][:20_000].cpu().numpy()
    rng = np.random.default_rng(3)
    keys = rng.choice(pool, n)
    x = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0
    y = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0 - x
    got = run_k6(keys, x, None, y, None, partition=True)
    calls = [c for c in launches.calls if c[0] == n]
    assert calls[0][2] == K.GROUPBY_PARTITIONS and calls[-1][2] == 0
    ones = np.ones(n, np.uint8)
    check_states(got, expected(keys, x, ones, y, ones))


def test_k6_rejects_an_untied_codev():
    v = torch.arange(10, dtype=torch.float64, device=DEV)
    w = v * 2
    k = torch.zeros(10, dtype=torch.int64, device=DEV)
    S, C, D, X = K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_CODEV_F64
    for vals, ops in (([v, w, None, v], [S, S, C, X]),   # no DEV of y after it
                      ([w, None, v, w], [S, C, X, D])):  # no SUM of x
        with pytest.raises(_lib.FugueB200KernelError, match="CODEV"):
            K.groupby_u64(k, None, vals, [None] * len(ops), ops, partition=False)


def test_k6_two_deviation_sets_of_one_column_both_sum():
    """Two DEV / DEV2 pairs naming the same column and validity each receive the full sums."""
    rng = np.random.default_rng(5)
    n = 50_000
    k = torch.from_numpy(rng.integers(0, 500, n)).to(DEV)
    v = torch.from_numpy(rng.normal(3.0, 2.0, n)).to(DEV)
    S, C, D, D2 = K.AGG_SUM_F64, K.AGG_COUNT, K.AGG_DEV_F64, K.AGG_DEV2_F64
    _, _, ga, _ = K.groupby_u64(k, None, [v, None, v, v, v, v], [None] * 6, [S, C, D, D2, D, D2], partition=False)
    assert torch.equal(ga[2], ga[4]) or torch.allclose(ga[2].view(torch.float64), ga[4].view(torch.float64),
                                                       rtol=0, atol=1e-9)
    assert torch.allclose(ga[3].view(torch.float64), ga[5].view(torch.float64), rtol=1e-12, atol=0)
    assert bool((ga[3].view(torch.float64) > 0).all())


@pytest.mark.parametrize("nulls", ["none", "x only"])
@pytest.mark.parametrize("pair_first", [False, True])
def test_pair_beside_variances_of_its_columns(nulls, pair_first):
    """CORR(x, y) with STDDEV(x) and VAR_POP(y) in one call: the variances share the pair's deviation sets where
    column and validity match, and neither side is lost."""
    from oracle import moments as OM

    rng = np.random.default_rng(6)
    n = 40_000
    x = rng.normal(10.0, 3.0, n)
    y = 0.5 * x + rng.normal(0.0, 1.0, n)
    xmask = rng.random(n) < 0.1 if nulls == "x only" else None
    tbl = pa.table({"k": rng.integers(0, 200, n), "x": pa.array(x, mask=xmask), "y": y})
    pair = {"r": f.corr(col("x"), col("y")), "b": f.regr_slope(col("y"), col("x"))}
    var = {"s": f.stddev(col("x")), "v": f.var_pop(col("y"))}
    aggs = {**pair, **var} if pair_first else {**var, **pair}
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, **aggs).as_arrow()
    groups: Dict[Any, List[dict]] = {}
    for r in tbl.to_pylist():
        groups.setdefault(r["k"], []).append(r)
    assert res.num_rows == len(groups)
    for r in res.to_pylist():
        rows = groups[r["k"]]
        pairs = OC.pair_rows([z["x"] for z in rows], [z["y"] for z in rows])
        check("CORR", r["r"], pairs, scan=False)
        check("REGR_SLOPE", r["b"], pairs, scan=False)
        for out, fn, vals in (("s", "STDDEV_SAMP", [z["x"] for z in rows if z["x"] is not None]),
                              ("v", "VAR_POP", [z["y"] for z in rows])):
            m = len(vals)
            ex = float(OM.exact_m2(vals))
            sx2 = float(sum(Fraction(v) ** 2 for v in vals))
            div = m - 1 if fn == "STDDEV_SAMP" else m
            var_ = ex / div
            tol = 2 * ((m + 2) * U * ex + (m * U) ** 2 * sx2) / div + 2 * U * var_  # the K6 bound of §7i
            got = r[out] ** 2 if fn == "STDDEV_SAMP" else r[out]
            assert abs(got - var_) <= tol + (4 * U * var_ if fn == "STDDEV_SAMP" else 0), (out, got, var_)


def test_shifted_data_and_the_textbook_formula_fails_the_same_bound():
    """Means 1e9, sigma 1e-3: the corrected two-pass stays within its bound; sum xy - sum x sum y / m does not."""
    rng = np.random.default_rng(9)
    ngroups, per = 100, 500
    keys = np.repeat(np.arange(ngroups, dtype=np.int64), per)
    x = 1e9 + rng.standard_normal(ngroups * per) * 1e-3
    y = 1e9 + (x - 1e9) * 0.7 + rng.standard_normal(ngroups * per) * 1e-3
    got = run_k6(keys, x, None, y, None, partition=False)
    ones = np.ones(len(x), np.uint8)
    want = expected(keys, x, ones, y, ones)
    check_states(got, want)
    fails = 0
    for k, pairs in want.items():
        a, b = np.array([p[0] for p in pairs]), np.array([p[1] for p in pairs])
        naive = float(np.sum(a * b) - np.sum(a) * np.sum(b) / len(a))
        st, e = errors(pairs, scan=False)
        fails += abs(naive - float(st[5])) > e[4]
    assert fails == ngroups


def test_k6_dyadic_4m_rows():
    """4 M rows, 65 536 keys, on the region path: exact integer sums of the reference."""
    rng = np.random.default_rng(4)
    n = 4_000_000
    keys = rng.integers(0, 65_536, n).astype(np.int64)
    kx = rng.integers(-(1 << 20) + 1, 1 << 20, n)
    ky = (kx // 3 + rng.integers(-(1 << 19), 1 << 19, n))
    xm = (rng.random(n) > 0.05).astype(np.uint8)
    got = run_k6(keys, kx / 1024.0, xm, ky / 1024.0, None, partition=True)
    want = OC.dyadic_group_states(keys, kx, ky, xm)
    for g, (m, mx, my, sxx, syy, sxy) in want.items():
        c, gmx, gmy, gxx, gyy, gxy = got[g]
        assert c == m
        # |x|, |y| < 2^10, so ||x||^2 <= m 2^20
        ex = 2 * ((m + 2) * U * float(sxx) + (m * U) ** 2 * m * 2.0 ** 20)
        ey = 2 * ((m + 2) * U * float(syy) + (m * U) ** 2 * m * 2.0 ** 20)
        exy = 2 * ((m + 2) * U * math.sqrt(float(sxx) * float(syy)) + (m * U) ** 2 * m * 2.0 ** 20)
        assert abs(gxx - float(sxx)) <= ex and abs(gyy - float(syy)) <= ey and abs(gxy - float(sxy)) <= exy, g
        assert abs(gmx - float(mx)) <= (m + 1) * U * 2.0 ** 10 and abs(gmy - float(my)) <= (m + 1) * U * 2.0 ** 10


# ---- engine calls on the hash path ---------------------------------------------------------------------
def test_edge_groups_through_aggregate():
    n = 20_000
    keys, x, xm, y, ym = edge_data(n, seed=1)
    tbl = pa.table({"k": keys, "x": pa.array(x, mask=xm == 0), "y": pa.array(y, mask=ym == 0)})
    aggs = {fn.lower(): build(fn, col("x"), col("y")) for fn in FUNCS}
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, **aggs).as_arrow()
    want = expected(keys, x, xm, y, ym)
    assert res.num_rows == len(want)
    for r in res.to_pylist():
        check_row(r, {fn.lower(): fn for fn in FUNCS}, want[r["k"]], scan=False)
    rows = {r["k"]: r for r in res.to_pylist()}
    c = rows[10**9]
    assert c["corr"] is None and c["regr_slope"] is None and c["regr_r2"] is None
    assert c["covar_pop"] == 0.0 and math.copysign(1.0, c["covar_pop"]) > 0
    assert rows[10**9 + 3]["regr_count"] == 0 and rows[10**9 + 3]["covar_pop"] is None
    assert rows[10**9 + 7]["regr_r2"] == 1.0 and rows[10**9 + 7]["corr"] is None


def test_empty_global_aggregate():
    tbl = pa.table({"k": pa.array([], pa.int64()), "x": pa.array([], pa.float64()), "y": pa.array([], pa.float64())})
    aggs = {fn.lower(): build(fn, col("x"), col("y")) for fn in FUNCS}
    want = {fn.lower(): (0 if fn == "REGR_COUNT" else None) for fn in FUNCS}
    for extra in ({}, {"m": f.median(col("x"))}):  # the hash route and the sorted route
        res = fa.aggregate(_df(tbl), None, engine=_engine(), as_fugue=True, **aggs, **extra).as_arrow()
        got = res.to_pylist()
        assert len(got) == 1 and {k: got[0][k] for k in want} == want
        assert res.schema.field("regr_count").type == pa.int64()
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, c=f.corr(col("x"), col("y"))).as_arrow()
    assert res.num_rows == 0


def test_more_than_16_accumulators_take_the_sorted_route(launches):
    rng = np.random.default_rng(11)
    n = 5000
    tbl = pa.table({"k": rng.integers(0, 20, n), "a": rng.standard_normal(n), "b": rng.standard_normal(n),
                    "c": rng.standard_normal(n)})
    res = fa.aggregate(_df(tbl), "k", engine=_engine(), as_fugue=True, p=f.corr(col("a"), col("b")),
                       q=f.covar_samp(col("a"), col("c"))).as_arrow()
    assert not any(c[0] == n for c in launches.calls)  # 24 accumulators: no hash group-by over the rows
    groups: Dict[Any, Any] = {}
    for r in tbl.to_pylist():
        groups.setdefault(r["k"], []).append(r)
    for r in res.to_pylist():
        rows = groups[r["k"]]
        check("CORR", r["p"], [(z["a"], z["b"]) for z in rows], scan=True)
        check("COVAR_SAMP", r["q"], [(z["a"], z["c"]) for z in rows], scan=True)


def test_matches_pandas_cov_and_corr():
    rng = np.random.default_rng(2)
    n = 30_000
    pdf = pd.DataFrame({"k": rng.integers(0, 300, n), "x": rng.normal(0, 10, n)})
    pdf["y"] = pdf["x"] * 0.3 + rng.normal(5, 2, n)
    res = fa.aggregate(pdf, "k", c=f.covar_samp(col("x"), col("y")), r=f.corr(col("x"), col("y")),
                       engine=_engine(), as_fugue=True).as_pandas().sort_values("k").reset_index(drop=True)
    g = pdf.groupby("k")
    assert np.allclose(res["c"], g.apply(lambda d: d["x"].cov(d["y"])).to_numpy(), rtol=1e-11, atol=0)
    assert np.allclose(res["r"], g.apply(lambda d: d["x"].corr(d["y"])).to_numpy(), rtol=1e-11, atol=0)


# ---- K9 co-moments scan ------------------------------------------------------------------------------
def scan_states(off: np.ndarray, x, xm, y, ym) -> List[Tuple]:
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    (res,) = K.segmented_comoments(t(off), len(x), [(t(x), t(xm), t(y), t(ym))])
    return res


def test_scan_at_tile_edges_and_across_tiles():
    rng = np.random.default_rng(7)
    lengths = [0, 1, 2, 3, 0, 2047, 2048, 2049, 5000, 1, 0, 777, 9000]
    n = sum(lengths)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    x = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0 + 1e6
    y = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 1024.0 - 0.25 * x
    x[rng.random(n) < 0.0005] = np.inf
    xm = (rng.random(n) > 0.1).astype(np.uint8)
    ym = (rng.random(n) > 0.1).astype(np.uint8)
    res = [r.cpu().tolist() for r in scan_states(off, x, xm, y, ym)]
    for a, b in zip(off[:-1], off[1:]):
        xs = [v if ok else None for v, ok in zip(x[a:b].tolist(), xm[a:b].tolist())]
        ys = [v if ok else None for v, ok in zip(y[a:b].tolist(), ym[a:b].tolist())]
        run = OC.running_states(xs, ys)
        for i, st in enumerate(run):
            assert res[0][a + i] == st[0]
            if st[0] == 0:
                assert all(res[j][a + i] == 0.0 for j in range(1, 6))
            elif i % 401 == 0 or i == b - a - 1 or i in (2046, 2047, 2048):
                got = {fn: None for fn in FUNCS}
                t = [torch.tensor([res[0][a + i]])] + [torch.tensor([res[j][a + i]], dtype=torch.float64)
                                                       for j in range(1, 6)]
                from fugue_b200.colmap import bivariate_of
                upto = OC.pair_rows(xs[:i + 1], ys[:i + 1])
                pre = errors(upto, True)
                for fn in FUNCS:
                    v, ok = bivariate_of(fn, *t)
                    got[fn] = v.item() if ok is None or ok.item() else None
                    check(fn, got[fn], upto, True, pre)


def test_scan_3m_rows_one_segment_bit_identical():
    rng = np.random.default_rng(12)
    n = 3_000_000
    kx = rng.integers(-(1 << 20) + 1, 1 << 20, n)
    ky = kx // 2 + rng.integers(-(1 << 19), 1 << 19, n)
    vm = (rng.random(n) > 0.03).astype(np.uint8)
    off = np.array([0, n], dtype=np.int64)
    first = scan_states(off, kx / 1024.0, vm, ky / 1024.0, None)
    again = scan_states(off, kx / 1024.0, vm, ky / 1024.0, None)
    for a, b in zip(first, again):
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    m, mx, my, sxx, syy, sxy = OC.dyadic_group_states(np.zeros(n, np.int64), kx, ky, vm)[0]
    got = [r[-1].item() for r in first]
    assert got[0] == m
    big = m * 2.0 ** 20  # ||x||^2, ||y||^2 <= m 2^20
    assert abs(got[3] - float(sxx)) <= 4 * m * U * math.sqrt(big * float(sxx))
    assert abs(got[4] - float(syy)) <= 4 * m * U * math.sqrt(big * float(syy))
    assert abs(got[5] - float(sxy)) <= 4 * m * U * math.sqrt(big) * max(math.sqrt(float(sxx)), math.sqrt(float(syy)))
    assert abs(got[1] - float(mx)) <= 4 * m * U * 2.0 ** 10 and abs(got[2] - float(my)) <= 4 * m * U * 2.0 ** 10


# ---- every engine call on every numeric storage type ---------------------------------------------------
TYPES = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(),
         pa.float16(), pa.float32(), pa.float64()]


def _typed_table(tp: pa.DataType, n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 50, n)
    y = (x // 2 + rng.integers(0, 25, n))
    k = rng.integers(0, 12, n)
    k[:5] = 99  # a group with one x value only: x constant
    x[:5] = 7
    return pa.table({"rid": np.arange(n), "k": k, "t": rng.permutation(n),
                     "x": pa.array(x, mask=rng.random(n) < 0.1).cast(tp),
                     "y": pa.array(y, mask=rng.random(n) < 0.1).cast(tp)})


def _groups(tbl: pa.Table, fx=lambda v: v, fy=lambda v: v) -> Dict[Any, List[Tuple[float, float]]]:
    out: Dict[Any, List[Tuple[float, float]]] = {}
    for r in tbl.to_pylist():
        out.setdefault(r["k"], [])
        if r["x"] is not None and r["y"] is not None:
            out[r["k"]].append((float(fx(r["x"])), float(fy(r["y"]))))
    return out


@pytest.mark.parametrize("tp", TYPES, ids=str)
def test_engine_calls_on_every_type(tp):
    tbl = _typed_table(tp, 3000, 3)
    e = _engine()
    names = {fn.lower(): fn for fn in FUNCS}
    aggs = {fn.lower(): build(fn, col("x"), col("y")) for fn in FUNCS}
    groups = _groups(tbl)
    # fa.aggregate (the hash route)
    res = fa.aggregate(_df(tbl), "k", engine=e, as_fugue=True, **aggs).as_arrow()
    assert res.num_rows == len(groups)
    for r in res.to_pylist():
        check_row(r, names, groups[r["k"]], scan=False)
    # a percentile in the same call: the sorted route
    res = fa.aggregate(_df(tbl), "k", engine=e, as_fugue=True, med=f.median(col("x")), **aggs).as_arrow()
    for r in res.to_pylist():
        check_row(r, names, groups[r["k"]], scan=True)
    # fa.select with expression arguments and HAVING
    sl = f.regr_slope(col("y") + 1, col("x") * 2)
    res = fa.select(_df(tbl), col("k"), sl.alias("s"), f.corr(col("x") * 2, col("y") + 1).alias("c"),
                    f.regr_count(col("y"), col("x")).alias("n"), having=f.regr_count(col("y"), col("x")) >= 150,
                    engine=e, as_fugue=True).as_arrow()
    g2 = _groups(tbl, lambda v: v * 2, lambda v: v + 1)
    assert res.num_rows == sum(len(p) >= 150 for p in groups.values())
    for r in res.to_pylist():
        assert r["n"] >= 150
        check("REGR_SLOPE", r["s"], g2[r["k"]], scan=False)
        check("CORR", r["c"], g2[r["k"]], scan=False)
    # raw SQL, REGR argument order included
    got = fa.raw_sql("SELECT k, CORR(x, y) AS c, COVAR_POP(x, y) AS p, regr_intercept(y, x) AS i, "
                     "REGR_AVGX(y, x) AS ax FROM", _df(tbl), "GROUP BY k ORDER BY k", engine=e,
                     as_fugue=True).as_arrow()
    for r in got.to_pylist():
        check_row(r, {"c": "CORR", "p": "COVAR_POP", "i": "REGR_INTERCEPT", "ax": "REGR_AVGX"}, groups[r["k"]], False)
    # ColumnMap windows: whole partition and running
    cols = [f.corr(col("x"), col("y")).over().alias("cw"), f.regr_slope(col("y"), col("x")).over().alias("sw"),
            f.regr_count(col("y"), col("x")).over(running=True).alias("nr"),
            f.covar_samp(col("x"), col("y")).over(running=True).alias("vr")]
    out = fa.transform(_df(tbl), ColumnMap("rid", *cols), schema="rid:long,cw:double,sw:double,nr:long,vr:double",
                       partition=PartitionSpec(by=["k"], presort="t"), engine=e, as_fugue=True).as_arrow()
    rows = {r["rid"]: r for r in tbl.to_pylist()}
    res = {r["rid"]: r for r in out.to_pylist()}
    parts: Dict[int, List[dict]] = {}
    for r in sorted(rows.values(), key=lambda r: r["t"]):
        parts.setdefault(r["k"], []).append(r)
    for key, prs in parts.items():
        allp = OC.pair_rows([r["x"] for r in prs], [r["y"] for r in prs])
        first = res[prs[0]["rid"]]
        check("CORR", first["cw"], allp, scan=True)
        check("REGR_SLOPE", first["sw"], allp, scan=True)
        for i, r in enumerate(prs):
            got = res[r["rid"]]
            assert (got["cw"], got["sw"]) == (first["cw"], first["sw"])  # the partition's value on every row
            if i % 37 == 0 or i == len(prs) - 1:
                upto = OC.pair_rows([z["x"] for z in prs[:i + 1]], [z["y"] for z in prs[:i + 1]])
                check("REGR_COUNT", got["nr"], upto, scan=True)
                check("COVAR_SAMP", got["vr"], upto, scan=True)


def test_window_residual_and_bit_identical_reruns():
    rng = np.random.default_rng(8)
    n = 30_000
    k = rng.integers(0, 4, n)  # partitions longer than a tile (2048 rows)
    x = rng.normal(10.0, 3.0, n)
    y = 2.0 * x + 1.0 + rng.normal(0, 0.5, n)
    tbl = pa.table({"rid": np.arange(n), "k": k, "t": rng.permutation(n), "x": x,
                    "y": pa.array(y, mask=rng.random(n) < 0.05)})
    resid = col("y") - (f.regr_intercept(col("y"), col("x")).over() + f.regr_slope(col("y"), col("x")).over() * col("x"))
    cols = [resid.alias("r"), f.regr_r2(col("y"), col("x")).over(running=True).alias("q")]

    def run():
        return fa.transform(_df(tbl), ColumnMap("rid", "k", "x", "y", *cols),
                            schema="rid:long,k:long,x:double,y:double,r:double,q:double",
                            partition=PartitionSpec(by=["k"], presort="t"), engine=_engine(), as_fugue=True).as_arrow()

    out = run()
    pdf = out.to_pandas()
    for key, g in pdf.groupby("k"):
        d = g.dropna(subset=["y"])
        slope, icept = np.polyfit(d["x"], d["y"], 1)
        assert np.allclose(d["r"], d["y"] - (icept + slope * d["x"]), rtol=0, atol=1e-9)
        assert g["r"].isna().sum() == g["y"].isna().sum()
    again = run()
    for c in ("r", "q"):
        assert np.array_equal(np.asarray(out.column(c).to_numpy(zero_copy_only=False)).view(np.int64),
                              np.asarray(again.column(c).to_numpy(zero_copy_only=False)).view(np.int64))


def test_rejections():
    tbl = pa.table({"k": [1, 2], "s": ["a", "b"], "b": [True, False], "v": [1.0, 2.0],
                    "d": pa.array([0, 1], pa.date32())})
    e = _engine()
    for arg in ("s", "b", "d"):
        with pytest.raises(NotImplementedError):
            fa.aggregate(_df(tbl), "k", engine=e, a=f.corr(col(arg), col("v")).alias("a"))
        with pytest.raises(NotImplementedError):
            fa.transform(_df(tbl), ColumnMap("k", f.corr(col("v"), col(arg)).over().alias("c")),
                         schema="k:long,c:double", partition=PartitionSpec(by=["k"]), engine=e)
    with pytest.raises(NotImplementedError):
        fa.select(_df(tbl), col("k"), f.corr(col("v"), col("v")).alias("c"), f.count_distinct(col("v")).alias("n"),
                  engine=e)
