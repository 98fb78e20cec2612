"""EWM_MEAN, EWM_VAR and EWM_STD on the H100 (``fb_segmented_ewm``, DESIGN §7s): the kernel against the exact reference
(oracle/ewm.py) row by row at tile edges, every position mode and both weightings; one 3 M-row partition (carry chunks)
and 65 536 partitions against pandas, with bit-identical reruns; every numeric storage type with NULL, NaN and +-inf;
time decay over timestamp, date32 and int64 order columns with ties and gaps; the ColumnMap, select / assign / filter
and SQL routes against ``pandas.groupby().ewm()``; and a spy showing one scan sequence per call."""
import datetime
import math
from decimal import Context, localcontext
from typing import Any, List

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
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
from oracle.ewm import ewm, ewm_sums  # noqa: E402

DEV = torch.device("cuda", 0)
_ENGINE: List[Any] = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


def _kernel(vals, offsets, alpha, adjust, pos, times=None, scale=1.0):
    v = torch.tensor([0.0 if x is None else x for x in vals], dtype=torch.float64, device=DEV)
    m = torch.tensor([x is not None for x in vals], dtype=torch.uint8, device=DEV)
    off = torch.tensor(offsets, dtype=torch.int64, device=DEV)
    t = None if times is None else torch.tensor(times, dtype=torch.int64, device=DEV)
    (res,) = K.segmented_ewm(off, len(vals), [(v, m, alpha, adjust, pos, t, scale, True)])
    return [x.cpu().numpy() for x in res]


def _close(got, ref, scale, rel=1e-12):
    return abs(got - ref) <= rel * (abs(ref) + scale)


def _check_sums(vals, offsets, alpha, adjust, ignore_na, times=None, halflife=None, decimal=False):
    """The kernel's count, mean, W, W2 and C on every row against the reference sums.  Without adjust the kernel keeps
    weight shares: W is 1 and W2, C are the reference's W2 / W^2 and C / W."""
    pos = K.EWM_TIMES if times is not None else (K.EWM_OBSERVATIONS if ignore_na else K.EWM_ROWS)
    cnt, mean, w, w2, c = _kernel(vals, offsets, alpha, adjust, pos, times, 1.0 / halflife if halflife else 1.0)
    with localcontext(Context(prec=60)):
        _check_rows(vals, offsets, alpha, adjust, ignore_na, times, halflife, decimal, cnt, mean, w, w2, c)


def _check_rows(vals, offsets, alpha, adjust, ignore_na, times, halflife, decimal, cnt, mean, w, w2, c):
    for a, b in zip(offsets, offsets[1:]):
        part = vals[a:b]
        ex = ewm_sums(part, alpha, adjust, ignore_na, None if times is None else times[a:b], halflife, decimal)
        lo, hi = math.inf, -math.inf
        for i, e in zip(range(a, b), ex):
            if vals[i] is not None and vals[i] == vals[i]:
                lo, hi = min(lo, vals[i]), max(hi, vals[i])
            if e is None:
                assert cnt[i] == 0 and mean[i] == 0 and c[i] == 0, i
                continue
            n, W, W2, S1, S2, _ = e
            assert cnt[i] == n, i
            m = S1 / W
            C = S2 - S1 * m
            if not adjust:
                W, W2, C = W / W, W2 / (W * W), C / W
            spread = max(hi - float(m), float(m) - lo)
            assert _close(mean[i], float(m), spread), (i, mean[i], float(m))
            assert _close(w[i], float(W), 0.0) and _close(w2[i], float(W2), 0.0), (i, w[i], float(W), w2[i], float(W2))
            if times is None:
                assert _close(c[i], float(C), float(W) * spread * (spread + abs(float(m)))), (i, c[i], float(C))


@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 4097])
@pytest.mark.parametrize("adjust, ignore_na", [(True, False), (False, False), (True, True), (False, True)])
def test_tile_edges_against_the_exact_reference(n, adjust, ignore_na):
    rng = np.random.default_rng(n)
    # dyadic alpha and values keep the exact sums small over one long partition
    vals = [None if rng.random() < 0.1 else float(rng.integers(-64, 64)) / 8 for _ in range(n)]
    _check_sums(vals, [0, n], 0.25, adjust, ignore_na)
    cuts = sorted(set(rng.integers(1, n, size=min(n - 1, 40)).tolist())) if n > 1 else []
    parts = [0] + cuts + [n]
    _check_sums(vals, parts, [0.1, 0.6, 1.0][n % 3], adjust, ignore_na)


def test_empty_and_tiny_partitions():
    vals = [None, 1.5, None, 2.0, 3.0, None, None, 4.0]
    _check_sums(vals, [0, 0, 1, 1, 3, 3, 6, 8], 0.3, False, False)
    assert [len(x) for x in _kernel([], [0], 0.3, True, K.EWM_ROWS)] == [0] * 5


def test_long_partition_with_gaps_without_adjust():
    # every other row NULL: pandas' running total T shrinks by beta + alpha = 0.3 + 0.7^2 at every gap, so the kernel
    # must not carry it
    rng = np.random.default_rng(41)
    n = 100_000
    vals = [None if i % 2 else float(rng.normal(1, 0.1)) for i in range(n)]
    _check_sums(vals, [0, n], 0.3, False, False, decimal=True)
    _check_sums(vals, [0, 40_001, n], 0.05, False, False, decimal=True)
    v = np.array([np.nan if x is None else x for x in vals])
    off = torch.tensor([0, n], dtype=torch.int64, device=DEV)
    (r,) = K.segmented_ewm(off, n, [(torch.from_numpy(v).to(DEV), None, 0.3, False, K.EWM_ROWS, None, 1.0, True)])
    cnt, mean, w, w2, c = (x.cpu().numpy() for x in r)
    s = pd.Series(v).ewm(alpha=0.3, adjust=False)
    assert np.allclose(mean, s.mean().to_numpy(), rtol=1e-11, atol=0)
    var = c / w * (w * w / (w * w - w2))
    assert np.allclose(var[2:], s.var().to_numpy()[2:], rtol=1e-8, atol=0)


def test_long_time_decay_without_adjust():
    # steps much shorter than the halflife, with ties: T grows by 0.5^(dt / 60) + 0.5 at every row
    rng = np.random.default_rng(42)
    n = 100_000
    ts = [int(x) for x in np.cumsum(rng.integers(0, 3, n))]
    vals = [None if rng.random() < 0.05 else float(rng.normal(3, 1)) for _ in range(n)]
    for adjust in (False, True):
        _check_sums(vals, [0, n], 0.5, adjust, False, times=ts, halflife=60)


def _pandas_rows(v: np.ndarray, offsets: np.ndarray, **kw) -> np.ndarray:
    k = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    df = pd.DataFrame({"k": k, "v": v})
    return df.groupby("k")["v"].ewm(**kw).mean().to_numpy()


def test_one_long_partition_and_bit_identical_reruns():
    rng = np.random.default_rng(11)
    n = 3_000_000
    v = rng.normal(5, 2, n)
    v[rng.random(n) < 0.05] = np.nan
    off = torch.tensor([0, n], dtype=torch.int64, device=DEV)
    col_ = (torch.from_numpy(v).to(DEV), None, 0.01, True, K.EWM_ROWS, None, 1.0, True)
    (a,) = K.segmented_ewm(off, n, [col_])
    (b,) = K.segmented_ewm(off, n, [col_])
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
    ref = pd.Series(v).ewm(alpha=0.01).mean().to_numpy()
    got = np.where(a[0].cpu().numpy() > 0, a[1].cpu().numpy(), np.nan)
    assert np.allclose(got, ref, rtol=1e-10, atol=1e-10, equal_nan=True)
    assert int(a[0][-1]) == int(np.sum(~np.isnan(v)))


def test_many_partitions_against_pandas():
    rng = np.random.default_rng(12)
    lengths = rng.integers(0, 40, 65_536)
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    n = int(offsets[-1])
    v = rng.normal(0, 3, n)
    v[rng.random(n) < 0.1] = np.nan
    off = torch.from_numpy(offsets).to(DEV)
    for adjust, ignore_na in ((True, False), (False, True)):
        pos = K.EWM_OBSERVATIONS if ignore_na else K.EWM_ROWS
        (r,) = K.segmented_ewm(off, n, [(torch.from_numpy(v).to(DEV), None, 0.2, adjust, pos, None, 1.0, False)])
        assert r[2] is None and r[3] is None and r[4] is None
        ref = _pandas_rows(v, offsets, alpha=0.2, adjust=adjust, ignore_na=ignore_na)
        got = np.where(r[0].cpu().numpy() > 0, r[1].cpu().numpy(), np.nan)
        assert np.allclose(got, ref, rtol=1e-12, atol=1e-12, equal_nan=True)


TYPES = {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "u8": pa.uint8(),
         "u16": pa.uint16(), "u32": pa.uint32(), "u64": pa.uint64(), "f16": pa.float16(), "f32": pa.float32(),
         "f64": pa.float64()}


def _typed_table(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    cols = {"rid": np.arange(n, dtype=np.int64), "k": rng.integers(0, 7, n), "t": rng.permutation(n)}
    for nm, tp in TYPES.items():
        if pa.types.is_floating(tp):
            x = rng.integers(-40, 40, n).astype(np.float64) / 4
            x[rng.random(n) < 0.04] = np.nan
            x[rng.random(n) < 0.01] = np.inf
            x[rng.random(n) < 0.01] = -np.inf
            arr = pa.array(x.astype(tp.to_pandas_dtype()) if tp != pa.float16() else x.astype(np.float16), type=tp,
                           mask=rng.random(n) < 0.1)
        else:
            lo, hi = (0, 100) if pa.types.is_unsigned_integer(tp) else (-100, 100)
            arr = pa.array(rng.integers(lo, hi, n), type=tp, mask=rng.random(n) < 0.1)
        cols[nm] = arr
    cols["c"] = np.full(n, 2.5)
    return pa.table(cols)


def _reference(tbl: pa.Table, nm: str, fn: str, alpha: float, adjust: bool = True, bias: bool = False) -> list:
    """Per input row, ``fn`` over its partition k in t order, by the exact reference."""
    k, t = tbl["k"].to_numpy(), tbl["t"].to_numpy()
    x = [None if v is None else float(v) for v in tbl[nm].to_pylist()]
    out: List[Any] = [None] * len(x)
    for key in np.unique(k):
        idx = np.flatnonzero(k == key)
        idx = idx[np.argsort(t[idx], kind="stable")]
        for i, r in zip(idx, ewm(fn, [x[j] for j in idx], alpha, adjust, bias=bias)):
            out[i] = r
    return out


def _same(got: list, ref: list, rel: float = 1e-11) -> None:
    for i, (g, r) in enumerate(zip(got, ref)):
        if r is None or g is None:
            assert g is None and r is None, (i, g, r)
        elif math.isnan(r) or math.isinf(r):
            assert (math.isnan(g) and math.isnan(r)) or g == r, (i, g, r)
        else:
            assert g == pytest.approx(r, rel=rel, abs=rel), (i, g, r)


@pytest.mark.parametrize("nm", list(TYPES))
def test_every_storage_type(nm):
    tbl = _typed_table(600, seed=len(nm) * 7 + ord(nm[-1]))
    spec = dict(partition_by=["k"], order_by=["t"])
    out = fa.select(_df(tbl), col("rid"), f.ewm_mean(nm, alpha=0.3).over(**spec).alias("m"),
                    f.ewm_var(nm, alpha=0.3, adjust=False).over(**spec).alias("v"),
                    f.ewm_std(nm, alpha=0.3, bias=True).over(**spec).alias("s"),
                    f.ewm_var("c", alpha=0.3).over(**spec).alias("z"), engine=_engine(), as_fugue=True).as_arrow()
    out = out.take(pc.sort_indices(out["rid"]))
    assert out.schema.field("m").type == pa.float64()
    _same(out["m"].to_pylist(), _reference(tbl, nm, "EWM_MEAN", 0.3))
    _same(out["v"].to_pylist(), _reference(tbl, nm, "EWM_VAR", 0.3, adjust=False), rel=1e-9)
    _same(out["s"].to_pylist(), _reference(tbl, nm, "EWM_STD", 0.3, bias=True), rel=1e-9)
    assert set(v for v in out["z"].to_pylist() if v is not None) == {0.0}  # constant runs: exactly 0


@pytest.mark.parametrize("tp, halflife, unit", [  # unit: storage units per step of t
    (pa.timestamp("s"), datetime.timedelta(minutes=3), 60), (pa.timestamp("ms"), datetime.timedelta(seconds=90), 1000),
    (pa.timestamp("us"), datetime.timedelta(hours=1), 3_600_000_000),
    (pa.timestamp("ns"), datetime.timedelta(microseconds=1500), 1_000_000), (pa.date32(), datetime.timedelta(days=2), 1),
    (pa.int64(), 2.5, 1), (pa.int32(), 7, 1)])
def test_time_decay(tp, halflife, unit):
    rng = np.random.default_rng(21)
    n = 3000
    k = rng.integers(0, 5, n)
    steps = rng.integers(0, 6, n) * (rng.random(n) < 0.9) + rng.integers(0, 50, n) * (rng.random(n) < 0.02)
    cum = np.cumsum(steps)
    t = cum * (unit if tp != pa.int64() and tp != pa.int32() else 1)  # ties and irregular gaps
    # tied rows may come in any order: give them one value (or NaN) so that no result depends on it
    v = np.sin(cum * 0.7) * 3
    v[cum % 11 == 3] = np.nan
    tcol = pa.array(t.astype(np.int32), type=pa.int32()).view(tp) if tp == pa.date32() else \
        pa.array(t, type=pa.int64()).cast(tp)
    tbl = pa.table({"rid": np.arange(n), "k": k, "t": tcol, "v": v})
    for adjust in (True, False):
        out = fa.transform(_df(tbl), ColumnMap("rid", f.ewm_mean(col("v"), halflife=halflife, times=True,
                                                                   adjust=adjust).alias("m")),
                           schema="rid:long,m:double", partition=PartitionSpec(by=["k"], presort="t"),
                           engine=_engine(), as_fugue=True).as_arrow()
        out = out.take(pc.sort_indices(out["rid"]))
        if isinstance(halflife, datetime.timedelta):  # the halflife in storage units of t
            us = halflife / datetime.timedelta(microseconds=1)
            h = us / 86_400_000_000 if tp == pa.date32() else us * {"s": 1e-6, "ms": 1e-3, "us": 1, "ns": 1e3}[tp.unit]
        else:
            h = halflife
        ref: List[Any] = [None] * n
        for key in range(5):
            idx = np.flatnonzero(k == key)
            r = ewm("EWM_MEAN", [None if np.isnan(x) else float(x) for x in v[idx]], 0.5, adjust,
                    times=[int(x) for x in t[idx]], halflife=h)
            for i, x in zip(idx, r):
                ref[i] = x
        _same(out["m"].to_pylist(), ref, rel=1e-10)


def test_time_decay_halflife_of_part_of_a_unit():
    # 12 hours over a date32 column: half a day, a fractional number of the column's units
    n = 500
    days = np.cumsum(np.random.default_rng(3).integers(0, 3, n)).astype(np.int32)
    v = np.sin(days * 0.3)
    tbl = pa.table({"rid": np.arange(n), "k": np.zeros(n, dtype=np.int64),
                    "t": pa.array(days, type=pa.int32()).view(pa.date32()), "v": v})
    out = fa.transform(_df(tbl), ColumnMap("rid", f.ewm_mean(col("v"), halflife=datetime.timedelta(hours=12),
                                                               times=True).alias("m")),
                       schema="rid:long,m:double", partition=PartitionSpec(by=["k"], presort="t"),
                       engine=_engine(), as_fugue=True).as_arrow()
    out = out.take(pc.sort_indices(out["rid"]))
    _same(out["m"].to_pylist(), ewm("EWM_MEAN", [float(x) for x in v], 0.5, times=[int(d) for d in days],
                                    halflife=0.5), rel=1e-10)
    ref = pd.Series(v).ewm(halflife=pd.Timedelta(hours=12), times=pd.to_datetime(days, unit="D")).mean()
    assert np.allclose(out["m"].to_numpy(), ref.to_numpy(), rtol=1e-10)


def test_time_decay_rejects_null_times_and_float_order():
    tbl = pa.table({"k": [1, 1, 1], "t": pa.array([1, None, 3], type=pa.int64()), "v": [1.0, 2.0, 3.0],
                    "tf": [1.0, 2.0, 3.0]})
    with pytest.raises(ValueError):
        fa.select(_df(tbl), f.ewm_mean("v", halflife=2, times=True).over(partition_by=["k"], order_by=["t"]).alias("m"),
                  engine=_engine(), as_fugue=True).as_arrow()
    with pytest.raises(ValueError):
        fa.select(_df(tbl), f.ewm_mean("v", halflife=2, times=True).over(partition_by=["k"], order_by=["tf"]).alias("m"),
                  engine=_engine(), as_fugue=True).as_arrow()


@pytest.mark.parametrize("bad", ["s", "b", "d"])
def test_non_numeric_arguments(bad):
    tbl = pa.table({"k": [1, 1], "t": [1, 2], "s": ["a", "b"], "b": [True, False],
                    "d": pa.array([1, 2], type=pa.date32())})
    with pytest.raises(NotImplementedError):
        fa.select(_df(tbl), f.ewm_mean(bad, alpha=0.5).over(partition_by=["k"], order_by=["t"]).alias("m"),
                  engine=_engine(), as_fugue=True).as_arrow()


def _routes_table(n: int = 5000) -> pa.Table:
    rng = np.random.default_rng(31)
    v = rng.normal(10, 4, n)
    v[rng.random(n) < 0.08] = np.nan
    return pa.table({"rid": np.arange(n), "k": rng.integers(0, 40, n), "t": rng.permutation(n), "v": v})


def _pandas(tbl: pa.Table, how: str, **kw) -> np.ndarray:
    df = tbl.to_pandas().sort_values(["k", "t"], kind="stable")
    g = df.groupby("k")["v"].ewm(**{k: v for k, v in kw.items() if k != "bias"})
    r = getattr(g, how)(**({"bias": kw["bias"]} if "bias" in kw else {}))
    return r.reset_index(level=0, drop=True).sort_index().to_numpy()


def test_routes_against_pandas_groupby():
    tbl = _routes_table()
    want = {"m": _pandas(tbl, "mean", alpha=0.2), "a": _pandas(tbl, "mean", com=3, adjust=False),
            "s": _pandas(tbl, "std", span=9, bias=False), "v": _pandas(tbl, "var", halflife=4, ignore_na=True),
            "p": _pandas(tbl, "mean", alpha=0.2, min_periods=3)}
    nodes = {"m": f.ewm_mean("v", alpha=0.2), "a": f.ewm_mean("v", com=3, adjust=False), "s": f.ewm_std("v", span=9),
             "v": f.ewm_var("v", halflife=4, ignore_na=True), "p": f.ewm_mean("v", alpha=0.2, min_periods=3)}
    spec = dict(partition_by=["k"], order_by=["t"])

    def check(out: pa.Table) -> None:
        out = out.take(pc.sort_indices(out["rid"]))
        for nm, ref in want.items():
            got = np.array([np.nan if x is None else x for x in out[nm].to_pylist()])
            assert np.allclose(got, ref, rtol=1e-11, atol=1e-11, equal_nan=True), nm

    check(fa.transform(_df(tbl), ColumnMap("rid", *[e.alias(nm) for nm, e in nodes.items()]),
                       schema="rid:long," + ",".join(f"{nm}:double" for nm in nodes),
                       partition=PartitionSpec(by=["k"], presort="t"), engine=_engine(), as_fugue=True).as_arrow())
    check(fa.select(_df(tbl), col("rid"), *[e.over(**spec).alias(nm) for nm, e in nodes.items()], engine=_engine(),
                    as_fugue=True).as_arrow())
    check(fa.assign(_df(tbl), engine=_engine(), as_fugue=True,
                    **{nm: e.over(**spec) for nm, e in nodes.items()}).as_arrow())
    kept = fa.filter(_df(tbl), f.ewm_mean("v", alpha=0.2).over(**spec) > 10, engine=_engine(),
                     as_fugue=True).as_arrow()
    assert sorted(kept["rid"].to_pylist()) == np.flatnonzero(want["m"] > 10).tolist()
    sql = fa.raw_sql("SELECT rid, EWM_MEAN(v, 0.2) OVER (PARTITION BY k ORDER BY t) AS m, "
                     "EWM_STD(v, 0.1, FALSE) OVER (PARTITION BY k ORDER BY t) AS s FROM", _df(tbl),
                     engine=_engine(), as_fugue=True).as_arrow()
    sql = sql.take(pc.sort_indices(sql["rid"]))
    for nm, ref in (("m", want["m"]), ("s", _pandas(tbl, "std", alpha=0.1, adjust=False))):
        got = np.array([np.nan if x is None else x for x in sql[nm].to_pylist()])
        assert np.allclose(got, ref, rtol=1e-11, atol=1e-11, equal_nan=True), nm


def test_one_scan_sequence_per_call(monkeypatch):
    calls: List[int] = []
    real = K.segmented_ewm

    def spy(off, n, columns):
        calls.append(len(columns))
        return real(off, n, columns)

    monkeypatch.setattr(K, "segmented_ewm", spy)
    tbl = _routes_table(3000)
    cm = ColumnMap("rid", f.ewm_mean(col("v"), alpha=0.2).alias("a"), f.ewm_var(col("v"), alpha=0.2).alias("b"),
                   f.ewm_std(col("v"), alpha=0.2, bias=True).alias("c"), f.ewm_mean(col("v"), com=2).alias("d"),
                   f.ewm_mean(col("v"), alpha=0.2, ignore_na=True).alias("e"))
    fa.transform(_df(tbl), cm, schema="rid:long,a:double,b:double,c:double,d:double,e:double",
                 partition=PartitionSpec(by=["k"], presort="t"), engine=_engine(), as_fugue=True).as_arrow()
    # a, b and c share one state column; d and e differ in their decay: three columns, one call
    assert calls == [3]
