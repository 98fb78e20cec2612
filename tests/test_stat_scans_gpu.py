"""The statistics scans of the window code on the H100 against the exact integer reference
(tests/_stat_scan_reference.py): ``fb_segmented_moments`` (VAR / STDDEV), ``fb_segmented_comoments`` (CORR / COVAR /
REGR_*) and ``fb_segmented_shape_moments`` (SKEWNESS / KURTOSIS), at the sizes where their shared tile and carry
kernels do something non-trivial: several warps of carry threads, carry threads that fold several tiles, segment
heads and empty segments on tile and carry-chunk starts (on all of them, and on every other one so that a carry
runs into each head), NULL-only tiles and carry chunks inside a segment, and
non-finite values on the row a partial last tile re-reads for its padding.  Then one window map per family through
``fa.transform`` above one carry pass of rows, checked with the suite's finishers and bounds."""
import math
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402
from oracle import moments as OM  # noqa: E402

import _stat_scan_reference as R  # noqa: E402
import test_comoments_gpu as TC  # noqa: E402 - the pair functions' finisher and bounds
import test_moments_gpu as TM  # noqa: E402 - the variances' finisher and bounds
import test_shape_moments_gpu as TS  # noqa: E402 - the shape statistics' finisher and bounds

DEV = torch.device("cuda", 0)
T = 2048  # rows per CTA of fb_segscan_tile_kernel (kTile)
# kCarryThreads of the scan traits in fb_window.cu: MomentScan 1024, CoMomentScan and ShapeScan 512.  A carry thread
# folds per = ceil(tiles / C) consecutive tiles, a carry chunk of per * T rows.
CARRY = {"moments": 1024, "comoments": 512, "shape_moments": 512}
SHAPES = ["singletons", "zipf", "spanning", "heads", "sparse_heads", "null_runs"]
NCOLS = K.SCAN_MAX_COLS + 1
SPECIAL = [math.inf, -math.inf, math.nan]
ALL_ROWS = 40_000  # below this every row is checked against its bound


def _sizes(c: int) -> List[int]:
    return [0, 1, T - 1, T, T + 1, 32 * T - 1, 32 * T + 1, c * T - 1, c * T, c * T + 1, 3 * c * T + 5]


CASES = [(fam, n) for fam, c in CARRY.items() for n in _sizes(c)]
MULTI = [(fam, n) for fam, n in CASES if n >= 32 * T + 1]


def _chunk(n: int, fam: str) -> int:
    """Rows per carry chunk."""
    ntiles = -(-n // T)
    return max(-(-ntiles // CARRY[fam]), 1) * T


# ---- data --------------------------------------------------------------------------------------------
def _offsets(n: int, fam: str, shape: str, rng: np.random.Generator) -> np.ndarray:
    if n == 0:
        return np.array([0, 0], dtype=np.int64)
    if shape == "singletons":
        return np.arange(n + 1, dtype=np.int64)
    if shape == "spanning":
        return np.array([0, n], dtype=np.int64)
    if shape == "zipf":  # Zipf-skewed lengths, and empty segments
        lens = np.zeros(0, np.int64)
        while lens.sum() < n:
            more = np.minimum(rng.zipf(1.3, n // 16 + 16), n)
            more[rng.random(len(more)) < 0.05] = 0
            lens = np.concatenate([lens, more])
        cut = np.concatenate([[0], np.cumsum(lens)])
        return np.concatenate([cut[cut < n], [n, n]]).astype(np.int64)
    if shape == "heads":  # a head on every tile start and carry-chunk start, empty segments stacked on some
        tiles = np.arange(0, n, T)
        chunks = np.arange(0, n, _chunk(n, fam))
        return np.sort(np.concatenate([tiles, tiles[::3], chunks, chunks, [n]])).astype(np.int64)
    if shape == "sparse_heads":  # heads on every other tile start and carry-chunk start, so that each head has
        # carried-in tiles next to it: the tile after a head and the chunk after a head take a carry that must stop
        # at that head
        tiles = np.arange(T, n, 2 * T)
        chunk = _chunk(n, fam)
        chunks = np.arange(0, n, 2 * chunk) if chunk > T else np.zeros(0, np.int64)
        return np.sort(np.concatenate([[0], tiles, tiles[::4], chunks, [n]])).astype(np.int64)
    if shape == "null_runs":  # one long segment, then one whose only valid row is its last (see _null_runs)
        return np.array([0, n - min(n, 3000), n], dtype=np.int64)
    raise ValueError(shape)


def _null_runs(n: int, fam: str, masks: List[np.ndarray]) -> None:
    """A whole tile of NULLs and a whole carry chunk of NULLs inside the first segment (in the first and the last
    of ``masks``: x and y of a pair), and the second segment valid on its last row only."""
    ntiles, chunk = -(-n // T), _chunk(n, fam)
    tail = n - min(n, 3000)
    t = ntiles // 3
    if (t + 1) * T <= tail:
        masks[0][t * T:(t + 1) * T] = 0
    j = 2 * (-(-n // chunk)) // 3
    if (j + 1) * chunk <= tail and j * chunk >= (t + 1) * T:
        masks[-1][j * chunk:(j + 1) * chunk] = 0
    for m in masks:
        m[tail:] = 0
    if n:
        masks[0][n - 1] = masks[-1][n - 1] = 1


def _special_rows(n: int, rng: np.random.Generator) -> np.ndarray:
    """The first row of the last tile (re-read for the padding of a partial tile), the first row of a tile three
    quarters in, and a few rows of the last quarter."""
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    ntiles = -(-n // T)
    rows = [(ntiles - 1) * T, (3 * ntiles // 4) * T]
    rows += rng.integers(3 * n // 4, n, 3).tolist()
    return np.unique(np.array(rows, dtype=np.int64))


def _column(fam: str, n: int, rng: np.random.Generator, i: int, special: bool) -> Dict[str, Any]:
    """Dyadic values of column (or pair) i with validity masks, and with ``special`` a few +-inf and NaN."""
    kmax = R.SHAPE_K if fam == "shape_moments" else R.MOMENT_K
    shift = R.SHAPE_SHIFT if fam == "shape_moments" else R.MOMENT_SHIFT
    k = rng.integers(-kmax + 1, kmax, n)
    c: Dict[str, Any] = {"x": R.dyadic(k, shift), "xv": (rng.random(n) > 0.1 + 0.05 * (i % 3)).astype(np.uint8)}
    if fam == "comoments":
        ky = np.clip(k // 2 + rng.integers(-(kmax // 2), kmax // 2, n), -kmax + 1, kmax - 1)
        c["y"] = R.dyadic(ky, -2.0 ** 19)
        c["yv"] = (rng.random(n) > 0.1).astype(np.uint8)
    if special:
        for side in ("x", "y") if fam == "comoments" else ("x",):
            rows = _special_rows(n, rng)
            if side == "y":  # independent of x's rows
                rows = np.unique(np.concatenate([rows[:1], rng.integers(n // 2, n, 2)])) if n else rows
            c[side][rows] = rng.choice(SPECIAL, len(rows))
            c[side + "v"][rows] = 1
    return c


def _apply_shape(fam: str, n: int, shape: str, cols: List[Dict[str, Any]]) -> None:
    """The NULL runs of ``shape`` in every column."""
    if shape == "null_runs":
        for c in cols:
            _null_runs(n, fam, [c["xv"], c["yv"]] if fam == "comoments" else [c["xv"]])


def _reference(fam: str, off: np.ndarray, c: Dict[str, Any]):
    if fam == "moments":
        return R.RunningMoments(off, c["x"], c["xv"])
    if fam == "shape_moments":
        return R.RunningShapeMoments(off, c["x"], c["xv"])
    return R.RunningCoMoments(off, c["x"], c["xv"], c["y"], c["yv"], R.MOMENT_SHIFT, -2.0 ** 19)


def _run(fam: str, off: np.ndarray, cols: List[Dict[str, Any]]) -> List[Tuple[torch.Tensor, ...]]:
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    n = len(cols[0]["x"])
    d_off = t(off)
    if fam == "comoments":
        res = K.segmented_comoments(d_off, n, [(t(c["x"]), t(c["xv"]), t(c["y"]), t(c["yv"])) for c in cols])
    else:
        run = K.segmented_moments if fam == "moments" else K.segmented_shape_moments
        res = run(d_off, n, [(t(c["x"]), t(c["xv"])) for c in cols])
    torch.cuda.synchronize()
    return [tuple(r) for r in res]


# ---- checks ------------------------------------------------------------------------------------------
def _checked_rows(n: int, fam: str, off: np.ndarray, rng: np.random.Generator) -> np.ndarray:
    """Every row of a small table; else every row within 3 of a tile or carry-chunk start, the first, second and
    last row of up to 3000 segments, and 20 000 random rows."""
    if n <= ALL_ROWS:
        return np.arange(n, dtype=np.int64)
    starts = np.concatenate([np.arange(0, n, T), np.arange(0, n, _chunk(n, fam))])
    near = (starts[:, None] + np.arange(-3, 4)).ravel()
    a, b = off[:-1], off[1:]
    keep = b > a
    a, b = a[keep], b[keep]
    pick = rng.choice(len(a), min(len(a), 3000), replace=False)
    a, b = a[pick], b[pick]
    rows = np.concatenate([near, a, np.minimum(a + 1, b - 1), b - 1, rng.integers(0, n, 20_000)])
    return np.unique(rows[(rows >= 0) & (rows < n)])


def _check(fam: str, ref, got: Tuple[torch.Tensor, ...], rows: np.ndarray, what: str) -> None:
    """The count on every row, exactly; every word 0 (+0.0) on every row where the count is 0; every word within its
    bound (or NaN / +-inf as the reference says) on ``rows``."""
    cnt, *words = got
    c = cnt.cpu().numpy()
    bad = np.flatnonzero(c != ref.count)
    assert len(bad) == 0, (what, "count", bad[:5], c[bad[:5]], ref.count[bad[:5]])
    empty = torch.from_numpy(ref.count == 0).to(DEV)
    for o, w in enumerate(words):
        nz = int((w.view(torch.int64)[empty] != 0).sum())
        assert nz == 0, (what, "word", o, "not +0.0 on", nz, "rows with no valid value")
    want, bound = ref.want(rows)
    idx = torch.from_numpy(rows).to(DEV)
    for o, (w, v, b) in enumerate(zip(words, want, bound)):
        g = w[idx].cpu().numpy()
        with np.errstate(invalid="ignore"):
            ok = (g == v) | (np.isnan(g) & np.isnan(v)) | (np.abs(g - v) <= b)
        if fam == "moments":
            ok &= ~(g < 0)
        fail = np.flatnonzero(~ok)
        assert len(fail) == 0, (what, "word", o, len(fail), "rows, first", rows[fail[:4]], g[fail[:4]], v[fail[:4]],
                                b[fail[:4]], ref.count[rows[fail[:4]]])


def _case_id(case: Tuple[str, int]) -> str:
    return f"{case[0]}-{case[1]}"


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_one_column_against_the_exact_reference(case, shape):
    fam, n = case
    rng = np.random.default_rng(n * 11 + SHAPES.index(shape) + 101 * len(fam))
    off = _offsets(n, fam, shape, rng)
    cols = [_column(fam, n, rng, 1, special=True)]
    _apply_shape(fam, n, shape, cols)
    (got,) = _run(fam, off, cols)
    _check(fam, _reference(fam, off, cols[0]), got, _checked_rows(n, fam, off, rng), f"{fam} n={n} {shape}")
    if n == 3 * CARRY[fam] * T + 5 and shape == "zipf":  # identical bits from run to run (fixed combination order)
        (again,) = _run(fam, off, cols)
        for a, b in zip(got, again):
            assert torch.equal(a.view(torch.int64), b.view(torch.int64))


@pytest.mark.parametrize("case", MULTI, ids=_case_id)
def test_more_columns_than_one_launch_against_the_exact_reference(case):
    """SCAN_MAX_COLS + 1 columns (two launch sequences) with different data and validity, column 0 without a mask,
    non-finite values in every other column; every column against the reference."""
    fam, n = case
    shape = SHAPES[MULTI.index(case) % len(SHAPES)]
    rng = np.random.default_rng(n * 13 + len(fam))
    off = _offsets(n, fam, shape, rng)
    cols = [_column(fam, n, rng, i, special=i % 2 == 1) for i in range(NCOLS)]
    _apply_shape(fam, n, shape, cols)
    cols[0]["xv"] = None
    if fam == "comoments":
        cols[0]["yv"] = None
    res = _run(fam, off, cols)
    assert len(res) == NCOLS
    rows = _checked_rows(n, fam, off, rng)
    for i, (c, got) in enumerate(zip(cols, res)):
        _check(fam, _reference(fam, off, c), got, rows, f"{fam} n={n} {shape} column {i}")


# ---- window maps through fa.transform ---------------------------------------------------------------
def _table(fam: str, n: int, rng: np.random.Generator) -> Tuple[pa.Table, Dict[str, Any]]:
    """n rows in one partition of C * T + 20 000 rows and a few thousand Zipf-sized ones, in random order, with
    dyadic values and about 15 % NULLs; also the columns as numpy arrays."""
    big = CARRY[fam] * T + 20_000
    key = np.concatenate([np.zeros(big, np.int64), np.minimum(rng.zipf(1.3, n - big), 3000)])
    key = key[rng.permutation(n)]
    c = _column(fam, n, rng, 1, special=False)
    data = {"rid": np.arange(n), "k": key, "t": rng.permutation(n)}
    for side in ("x", "y") if fam == "comoments" else ("x",):
        data[side] = pa.array(c[side], mask=c[side + "v"] == 0)
    return pa.table(data), {"k": key, "t": data["t"], **c}


def _transform(tbl: pa.Table, cols: List[Any]) -> Dict[str, Any]:
    """Per output column, (value or None) per rid."""
    schema = "rid:long," + ",".join(f"{c.output_name}:double" for c in cols)
    out = fa.transform(B200DataFrame(B200Table.from_arrow(tbl, DEV)), ColumnMap("rid", *cols), schema=schema,
                       partition=PartitionSpec(by=["k"], presort="t"), engine=TM._engine(), as_fugue=True).as_arrow()
    rid = out.column("rid").to_numpy()
    res: Dict[str, Any] = {}
    for c in cols:
        a = out.column(c.output_name)
        v = np.empty(len(rid))
        null = np.zeros(len(rid), bool)
        v[rid] = a.to_numpy(zero_copy_only=False)
        null[rid] = a.is_null().to_numpy(zero_copy_only=False)
        res[c.output_name] = (v, null)
    return res


def _sorted(data: Dict[str, Any], sides: Tuple[str, ...]):
    """The rows in partition order (key, then t): the order, the partition offsets and the reordered columns."""
    order = np.lexsort((data["t"], data["k"]))
    k = data["k"][order]
    off = np.concatenate([[0], np.flatnonzero(k[1:] != k[:-1]) + 1, [len(k)]]).astype(np.int64)
    cols = {s: data[s][order] for s in sides}
    cols.update({s + "v": data[s + "v"][order] for s in sides})
    return order, off, cols


def _sample(off: np.ndarray, rng: np.random.Generator) -> List[Tuple[int, int]]:
    """(position, last position of its partition): the first, second and last row of 300 partitions and of the
    largest, and 1500 random rows of the largest."""
    a, b = off[:-1], off[1:] - 1
    big = int(np.argmax(b - a))
    pick = np.unique(np.concatenate([rng.choice(len(a), min(300, len(a)), replace=False), [big]]))
    out = [(int(p), int(b[s])) for s in pick for p in {a[s], min(a[s] + 1, b[s]), b[s]}]
    out += [(int(p), int(b[big])) for p in rng.integers(a[big], b[big] + 1, 1500)]
    return out


def _got(res: Dict[str, Any], name: str, rid: int) -> Optional[float]:
    v, null = res[name]
    return None if null[rid] else float(v[rid])


def test_variance_window_map_above_one_carry_pass():
    rng = np.random.default_rng(21)
    tbl, data = _table("moments", 2_200_000, rng)
    cols = [f.var_samp(col("x")).over(running=True).alias("vr"), f.var_samp(col("x")).over().alias("vw"),
            f.stddev_pop(col("x")).over(running=True).alias("sr"), f.stddev_pop(col("x")).over().alias("sw")]
    res = _transform(tbl, cols)
    order, off, c = _sorted(data, ("x",))
    ref = R.RunningMoments(off, c["x"], c["xv"])

    def check(fn: str, got: Optional[float], p: int) -> None:
        m = int(ref.count[p])
        if OM.result(fn, m, 0.0) is None:
            assert got is None, (fn, p, got)
            return
        assert got is not None, (fn, p, m)
        (_,), (b,) = ref.want(np.array([p]))
        TM.check_finite_result(fn, got, m, ref.m2_fraction(p), float(b[0]))

    for p, last in _sample(off, rng):
        rid = int(order[p])
        check("VAR_SAMP", _got(res, "vr", rid), p)
        check("STDDEV_POP", _got(res, "sr", rid), p)
        check("VAR_SAMP", _got(res, "vw", rid), last)
        check("STDDEV_POP", _got(res, "sw", rid), last)


def test_pair_window_map_above_one_carry_pass():
    rng = np.random.default_rng(22)
    tbl, data = _table("comoments", 1_100_000, rng)
    x, y = col("x"), col("y")
    cols = [TC.build("COVAR_SAMP", x, y).over(running=True).alias("cr"),
            TC.build("CORR", x, y).over(running=True).alias("rr"),
            TC.build("REGR_SLOPE", x, y).over().alias("sw")]
    res = _transform(tbl, cols)
    order, off, c = _sorted(data, ("x", "y"))
    ref = R.RunningCoMoments(off, c["x"], c["xv"], c["y"], c["yv"], R.MOMENT_SHIFT, -2.0 ** 19)
    for p, last in _sample(off, rng):
        rid = int(order[p])
        run, whole = (ref.state(p), ref.errors(p)), (ref.state(last), ref.errors(last))
        TC.check("COVAR_SAMP", _got(res, "cr", rid), (), True, run)
        TC.check("CORR", _got(res, "rr", rid), (), True, run)
        TC.check("REGR_SLOPE", _got(res, "sw", rid), (), True, whole)


def test_shape_window_map_above_one_carry_pass():
    rng = np.random.default_rng(23)
    tbl, data = _table("shape_moments", 1_100_000, rng)
    cols = [f.skewness(col("x")).over().alias("sw"), f.kurtosis(col("x")).over(running=True).alias("kr")]
    res = _transform(tbl, cols)
    order, off, c = _sorted(data, ("x",))
    ref = R.RunningShapeMoments(off, c["x"], c["xv"])
    for p, last in _sample(off, rng):
        rid = int(order[p])
        TS.check_finished("SKEWNESS", _got(res, "sw", rid), ref.central_sums(last), lambda: ref.bounds(last))
        TS.check_finished("KURTOSIS", _got(res, "kr", rid), ref.central_sums(p), lambda: ref.bounds(p))
