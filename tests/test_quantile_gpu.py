"""PERCENTILE_CONT / PERCENTILE_DISC / MEDIAN on the H100 (K10), bit for bit against ``oracle/quantile.py``: the
kernel on both paths and at their edges, the engine's aggregate / select / SQL, and the window form in
``fa.transform``."""
import math
import struct
from collections import OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema, type_to_expr
from fugue_b200.table import B200Table
from oracle import quantile as Q
from oracle import window as W
from oracle.keys import canonical_rows

DEV = torch.device("cuda", 0)
T = K.QUANTILE_TILE_ROWS
CLS = {"I64": (K.RANGE_KEY_I64, pa.int64()), "U64": (K.RANGE_KEY_U64, pa.uint64()),
       "F64": (K.RANGE_KEY_F64, pa.float64())}
_ENGINE = []


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


# ---- the kernel ------------------------------------------------------------------------------------------
def _values(rng, n, cls, null_rate=0.1):
    if cls == "F64":
        special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, 1e308, -1e308])
        v = np.where(rng.random(n) < 0.15, rng.choice(special, n), np.round(rng.standard_normal(n) * 40) / 8)
    elif cls == "U64":
        v = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
        v[rng.random(n) < 0.3] = np.uint64((1 << 63) + 5)
    else:
        v = rng.integers(-(1 << 63), 1 << 63, n, dtype=np.int64)
        small = rng.random(n) < 0.5  # ties
        v[small] = rng.integers(-3, 3, int(small.sum()))
    mask = rng.random(n) < null_rate
    return v, mask


def _check_kernel(values, mask, offsets, cls, qs):
    """Run the kernel and compare with the oracle, every segment, every q."""
    code, tp = CLS[cls]
    arr = pa.array(values, type=tp, mask=mask if mask is not None and mask.any() else None)
    tbl = pa.table({"v": arr})
    store = torch.from_numpy(np.ascontiguousarray(values).view(np.int64) if cls != "F64" else
                             np.ascontiguousarray(values, dtype=np.float64)).to(DEV)
    valid = None if mask is None else torch.from_numpy((~mask).astype(np.uint8)).to(DEV)
    off = torch.from_numpy(np.asarray(offsets, dtype=np.int64)).to(DEV)
    kinds = [(q, K.QUANTILE_CONT if k == Q.CONT else K.QUANTILE_DISC) for q, k in qs]
    count, outs = K.segmented_quantile(off, store, valid, code, kinds)
    m_exp, res_exp = Q.segment_quantiles(tbl, "v", np.asarray(offsets), qs)
    assert np.array_equal(count.cpu().numpy(), m_exp)
    for (q, k), o, exp in zip(qs, outs, res_exp):
        got = o.cpu().numpy()
        if k == Q.CONT:
            want = np.array([0.0 if x is None else x for x in exp], dtype=np.float64)
            bad = np.nonzero(got.view(np.int64) != want.view(np.int64))[0]
        else:
            want = np.array([-1 if x is None else x for x in exp], dtype=np.int64)
            bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, (cls, q, k, bad[:5], got[bad[:5]], want[bad[:5]])


QS = [(0.0, Q.CONT), (0.5, Q.CONT), (0.9, Q.CONT), (1.0, Q.CONT), (0.0, Q.DISC), (0.5, Q.DISC), (0.99, Q.DISC),
      (1.0, Q.DISC)]


def _offsets_of(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


@pytest.mark.parametrize("cls", ["I64", "U64", "F64"])
@pytest.mark.parametrize("nulls", [False, True])
def test_kernel_segment_lengths_at_the_tile_edges(cls, nulls):
    rng = np.random.default_rng(len(cls) * 7 + nulls)
    lengths = np.array([0, 1, 2, T - 1, T, T + 1, 2 * T] * 3)
    rng.shuffle(lengths)
    off = _offsets_of(lengths)
    v, mask = _values(rng, int(off[-1]), cls)
    _check_kernel(v, mask if nulls else None, off, cls, QS)


def test_kernel_window_edges_and_mixed_paths():
    rng = np.random.default_rng(3)
    # a T-row segment starting on the last row of window 0; T and T + 1 adjacent; a long segment (covering a
    # window in which no segment starts) between short ones; trailing empty segments
    lengths = [T - 1, T, T, T + 1, 5, 3 * T + 7, 9, 1, T + 1, T, 0, 0]
    off = _offsets_of(lengths)
    v, mask = _values(rng, int(off[-1]), "F64")
    _check_kernel(v, mask, off, "F64", QS)
    _check_kernel(rng.integers(-9, 9, int(off[-1])), None, off, "I64", QS)


def test_kernel_many_short_segments_and_16_quantiles():
    rng = np.random.default_rng(11)
    lengths = rng.integers(0, 40, 20_000)
    off = _offsets_of(lengths)
    v, mask = _values(rng, int(off[-1]), "F64")
    qs = [(float(q), Q.CONT if i % 2 else Q.DISC) for i, q in enumerate(np.linspace(0, 1, 16))]
    _check_kernel(v, mask, off, "F64", qs)
    _check_kernel(v, mask, off, "F64", qs + [(0.37, Q.CONT)])  # 17: two calls


def test_kernel_special_segments():
    inf = np.inf
    segs = [[np.nan] * 5, [np.nan, -np.nan, np.nan], [1.0, 2.0, inf], [-inf, inf], [-0.0, 0.0], [0.0, -0.0],
            [5.0] * 7, [inf, inf, -inf], [3.0], [], [2.0, np.nan, 1.0]]
    v = np.array([x for s in segs for x in s], dtype=np.float64)
    off = _offsets_of([len(s) for s in segs])
    mask = np.zeros(len(v), dtype=bool)
    mask[-2] = True  # a NULL in the middle of a segment
    _check_kernel(v, mask, off, "F64", QS)
    allnull = np.ones(len(v), dtype=bool)
    _check_kernel(v, allnull, off, "F64", QS)
    # the same shapes, long
    big = np.concatenate([np.full(T + 3, np.nan), np.full(T + 5, 5.0), np.where(np.arange(3 * T) % 2, -0.0, 0.0)])
    _check_kernel(big, None, _offsets_of([T + 3, T + 5, 3 * T]), "F64", QS)
    u = np.array([(1 << 64) - 1, 1 << 63, 0, (1 << 63) - 1, 12], dtype=np.uint64)
    _check_kernel(u, None, _offsets_of([5]), "U64", QS)
    _check_kernel(np.tile(u, T), None, _offsets_of([5 * T]), "U64", QS)


def test_kernel_empty_table():
    _check_kernel(np.zeros(0), None, np.array([0, 0, 0]), "F64", QS)
    count, outs = K.segmented_quantile(torch.zeros(1, dtype=torch.int64, device=DEV),
                                       torch.zeros(0, dtype=torch.float64, device=DEV), None, K.RANGE_KEY_F64,
                                       [(0.5, K.QUANTILE_CONT)])
    assert count.numel() == 0 and outs[0].numel() == 0


def test_kernel_one_3m_row_segment():
    rng = np.random.default_rng(5)
    n = 3_000_000
    v = rng.integers(-1000, 1000, n)
    mask = rng.random(n) < 0.05
    _check_kernel(v, mask, np.array([0, n]), "I64", QS)
    x = rng.standard_normal(n)
    _check_kernel(x, None, np.array([0, 7, n - 9, n]), "F64", QS)


def test_kernel_runs_are_identical():
    rng = np.random.default_rng(8)
    off = torch.from_numpy(_offsets_of(rng.integers(0, 3 * T, 300))).to(DEV)
    v = torch.from_numpy(rng.standard_normal(int(off[-1]))).to(DEV)
    a = K.segmented_quantile(off, v, None, K.RANGE_KEY_F64, [(0.3, K.QUANTILE_CONT), (0.7, K.QUANTILE_DISC)])
    b = K.segmented_quantile(off, v, None, K.RANGE_KEY_F64, [(0.3, K.QUANTILE_CONT), (0.7, K.QUANTILE_DISC)])
    assert torch.equal(a[0], b[0]) and all(torch.equal(x.view(torch.int64), y.view(torch.int64))
                                           for x, y in zip(a[1], b[1]))


# ---- the engine ------------------------------------------------------------------------------------------
def _df(tbl):
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


def _by_key(res: pa.Table, keys):
    rows = canonical_rows(res, keys) if keys else [()] * res.num_rows
    assert len(set(rows)) == len(rows), "a group came out twice"
    return {k: i for i, k in enumerate(rows)}


def _same(got, want, kind):
    if want is None:
        return got is None
    if kind == Q.CONT:
        return got is not None and (_bits(got) == _bits(want) or (math.isnan(got) and math.isnan(want)))
    if isinstance(want, float) and math.isnan(want):
        return isinstance(got, float) and math.isnan(got)
    return got == want and (not isinstance(want, float) or math.copysign(1, got) == math.copysign(1, want))


def _check_groups(tbl, res, keys, specs):
    """``specs``: (output name, column, q, kind) per quantile column of ``res``."""
    at = _by_key(res, keys)
    groups = Q.group_rows(tbl, keys)
    assert set(at) == set(groups)
    for out, name, q, kind in specs:
        vals = tbl.column(name).to_pylist()
        got = res.column(out).to_pylist()
        exp = Q.group_quantiles(tbl, keys, name, [(q, kind)])
        for k, i in at.items():
            r = exp[k][1][0]
            want = r if kind == Q.CONT or r is None else vals[r]
            assert _same(got[i], want, kind), (out, k, got[i], want)


def _table(rng, n, ngroups=50):
    return pa.table({
        "k": pa.array(rng.integers(0, ngroups, n), mask=rng.random(n) < 0.05),
        "s": pa.array(rng.choice(["a", "bb", "c", "zz"], n), mask=rng.random(n) < 0.05),
        "fk": pa.array(rng.choice([0.0, -0.0, np.nan, 1.5, -2.0], n)),
        "v": pa.array(np.round(rng.standard_normal(n) * 100) / 4, mask=rng.random(n) < 0.1),
        "i": pa.array(rng.integers(-50, 50, n).astype(np.int32), mask=rng.random(n) < 0.1),
        "u": pa.array(rng.integers(0, 1 << 64, n, dtype=np.uint64), type=pa.uint64()),
        "h": pa.array(rng.standard_normal(n).astype(np.float16)),
        "b": pa.array(rng.random(n) < 0.5),
        "d": pa.array(rng.integers(0, 20000, n).astype(np.int32), type=pa.int32()).cast(pa.date32()),
        "ts": pa.array(rng.integers(0, 10**12, n), type=pa.int64()).view(pa.timestamp("us")),
        "str": pa.array(rng.choice(["x", "yy", "a", "", "é"], n), mask=rng.random(n) < 0.1),
    })


@pytest.mark.parametrize("keys", [[], ["k"], ["k", "s"], ["s"], ["fk"]])
def test_aggregate_every_key_shape(keys):
    rng = np.random.default_rng(len(keys) * 3 + len("".join(keys)))
    tbl = _table(rng, 20_000)
    aggs = dict(m=f.median(col("v")), p9=f.percentile_cont(col("i"), 0.9), pu=f.percentile_cont(col("u"), 0.25),
                ph=f.percentile_cont(col("h"), 0.75), dv=f.percentile_disc(col("v"), 0.3),
                ds=f.percentile_disc(col("str"), 0.5), dd=f.percentile_disc(col("d"), 0.8),
                dt=f.percentile_disc(col("ts"), 0.1), db=f.percentile_disc(col("b"), 0.5),
                di=f.percentile_disc(col("i"), 1))
    res = fa.aggregate(_df(tbl), partition_by=keys or None, **aggs, engine=_engine(), as_fugue=True).as_arrow()
    assert res.schema.field("m").type == pa.float64() and res.schema.field("ds").type == pa.string()
    assert res.schema.field("dd").type == pa.date32() and res.schema.field("dt").type == pa.timestamp("us")
    assert res.schema.field("di").type == pa.int32() and res.schema.field("db").type == pa.bool_()
    _check_groups(tbl, res, keys, [("m", "v", 0.5, Q.CONT), ("p9", "i", 0.9, Q.CONT), ("pu", "u", 0.25, Q.CONT),
                                   ("ph", "h", 0.75, Q.CONT), ("dv", "v", 0.3, Q.DISC), ("ds", "str", 0.5, Q.DISC),
                                   ("dd", "d", 0.8, Q.DISC), ("dt", "ts", 0.1, Q.DISC), ("db", "b", 0.5, Q.DISC),
                                   ("di", "i", 1.0, Q.DISC)])


def test_aggregate_next_to_the_other_aggregates():
    rng = np.random.default_rng(2)
    tbl = _table(rng, 30_000, 300)
    res = fa.aggregate(_df(tbl), "k", m=f.median(col("v")), s=f.sum(col("v")), c=f.count(col("v")),
                       n=f.count(col("*")), a=f.avg(col("i")), lo=f.min(col("i")), hi=f.max(col("v")),
                       fi=f.first(col("str")), la=f.last(col("v")), engine=_engine(), as_fugue=True).as_arrow()
    ref = fa.aggregate(_df(tbl), "k", s=f.sum(col("v")), c=f.count(col("v")), n=f.count(col("*")),
                       a=f.avg(col("i")), lo=f.min(col("i")), hi=f.max(col("v")), fi=f.first(col("str")),
                       la=f.last(col("v")), engine=_engine(), as_fugue=True).as_arrow()
    at, rat = _by_key(res, ["k"]), _by_key(ref, ["k"])
    assert set(at) == set(rat)
    for name in ["c", "n", "lo", "hi", "fi", "la"]:
        g, r = res.column(name).to_pylist(), ref.column(name).to_pylist()
        assert all(g[at[k]] == r[rat[k]] for k in at), name
    for name in ["s", "a"]:
        g, r = res.column(name).to_pylist(), ref.column(name).to_pylist()
        assert all((g[at[k]] is None and r[rat[k]] is None) or math.isclose(g[at[k]], r[rat[k]], rel_tol=1e-12,
                                                                               abs_tol=1e-9) for k in at), name
    assert res.schema == pa.schema([("k", pa.int64()), ("m", pa.float64())] + [(n, ref.schema.field(n).type)
                                                                                for n in ref.schema.names[1:]])
    _check_groups(tbl, res, ["k"], [("m", "v", 0.5, Q.CONT)])


def test_aggregate_empty_table():
    tbl = _table(np.random.default_rng(0), 0)
    res = fa.aggregate(_df(tbl), m=f.median(col("v")), d=f.percentile_disc(col("str"), 0.5), c=f.count(col("*")),
                       engine=_engine(), as_fugue=True).as_arrow()
    assert res.to_pylist() == [{"m": None, "d": None, "c": 0}]
    assert res.schema.field("d").type == pa.string()
    res = fa.aggregate(_df(tbl), "k", m=f.median(col("v")), engine=_engine(), as_fugue=True).as_arrow()
    assert res.num_rows == 0


def test_aggregate_above_the_partitioned_group_by_size():
    rng = np.random.default_rng(9)
    n = K.GROUPBY_PARTITION_MIN_ROWS + 1000
    k = rng.integers(0, 100, n)
    v = rng.standard_normal(n)
    tbl = pa.table({"k": k, "v": v})
    res = fa.aggregate(_df(tbl), "k", m=f.median(col("v")), p=f.percentile_cont(col("v"), 0.99),
                       engine=_engine(), as_fugue=True).as_arrow().to_pandas().set_index("k").sort_index()
    want = pd.DataFrame({"k": k, "v": v}).groupby("k")["v"]
    assert np.array_equal(res.m.to_numpy().view(np.int64), want.quantile(0.5).to_numpy().view(np.int64))
    assert np.array_equal(res.p.to_numpy().view(np.int64), want.quantile(0.99).to_numpy().view(np.int64))


def test_select_where_having_and_expressions():
    rng = np.random.default_rng(4)
    tbl = _table(rng, 20_000)
    e = _engine()
    med = f.median(col("v"))
    res = fa.select(_df(tbl), col("k"), med.alias("m"), (f.median(col("v") * 2) - med).alias("x"),
                    f.sum(col("i")).alias("s"), f.percentile_disc(col("str"), 0.5).alias("d"),
                    where=col("i") > -40, having=med > 1, engine=e, as_fugue=True).as_arrow()
    flt = tbl.filter(pa.compute.fill_null(pa.compute.greater(tbl.column("i"), -40), False))
    exp = Q.group_quantiles(flt, ["k"], "v", [(0.5, Q.CONT)])
    want = {k: r[1][0] for k, r in exp.items() if r[1][0] is not None and r[1][0] > 1}
    at = _by_key(res, ["k"])
    assert set(at) == set(want)
    m, x = res.column("m").to_pylist(), res.column("x").to_pylist()
    for k, i in at.items():
        assert _bits(m[i]) == _bits(want[k])
        assert x[i] == want[k]  # median(2v) = 2 median(v) exactly, for these values


def test_select_rejects_count_distinct_with_a_quantile():
    tbl = _table(np.random.default_rng(1), 100)
    with pytest.raises(NotImplementedError):
        fa.select(_df(tbl), col("k"), f.median(col("v")).alias("m"), f.count_distinct(col("i")).alias("c"),
                  engine=_engine())


@pytest.mark.parametrize("sql", ["MEDIAN(v)", "PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY v)",
                                 "PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY v ASC)", "QUANTILE_CONT(v, 0.5)"])
def test_raw_sql_spellings(sql):
    rng = np.random.default_rng(6)
    n = 50_000
    pdf = pd.DataFrame({"key": rng.integers(0, 200, n), "v": rng.standard_normal(n), "w": rng.integers(0, 9, n)})
    got = fa.raw_sql(f"SELECT key, {sql} AS m, PERCENTILE_DISC(0.9) WITHIN GROUP (ORDER BY w) AS d, "
                     "QUANTILE_DISC(w, 0.2) AS d2, COUNT(*) AS c FROM", pdf,
                     "WHERE w > 0 GROUP BY key HAVING MEDIAN(v) > -0.5 ORDER BY key", engine=_engine(), as_local=True)
    flt = pdf[pdf.w > 0]
    g = flt.groupby("key")
    want = pd.DataFrame({"m": g.v.quantile(0.5), "d": g.w.quantile(0.9, interpolation="higher"), "c": g.size()})
    want["d2"] = g.w.apply(lambda s: np.quantile(s.to_numpy(), 0.2, method="inverted_cdf"))
    want["d"] = g.w.apply(lambda s: np.quantile(s.to_numpy(), 0.9, method="inverted_cdf"))
    want = want[want.m > -0.5].reset_index()
    assert np.array_equal(got.key.to_numpy(), want.key.to_numpy())
    assert np.array_equal(got.m.to_numpy().view(np.int64), want.m.to_numpy().view(np.int64))
    assert np.array_equal(got.d.to_numpy(), want.d.to_numpy()) and np.array_equal(got.d2.to_numpy(), want.d2.to_numpy())
    assert np.array_equal(got.c.to_numpy(), want.c.to_numpy())


def test_window_forms_are_rejected_by_select():
    tbl = _table(np.random.default_rng(1), 10)
    with pytest.raises(NotImplementedError):
        fa.select(_df(tbl), f.median(col("v")).over().alias("m"), engine=_engine())


# ---- the window form -------------------------------------------------------------------------------------
def _run_map(tbl, cols, by, presort, algo):
    sch = Schema(tbl.schema)
    fields = [("rid", pa.int64())] + [(c.output_name, c.infer_type(sch) or pa.float64()) for c in cols]
    spec = PartitionSpec(by=by, algo=algo, **({"presort": presort} if presort else {}))
    return fa.transform(_df(tbl), ColumnMap("rid", *cols),
                        schema=",".join(f"{n}:{type_to_expr(t)}" for n, t in fields), partition=spec,
                        engine=_engine(), as_fugue=True).as_arrow()


@pytest.mark.parametrize("algo", ["hash", "even", "rand"])
@pytest.mark.parametrize("presort", [None, "rid desc"])
@pytest.mark.parametrize("keys", [["k"], ["s", "fk"], []])
def test_window_median_and_disc_in_transform(algo, presort, keys):
    rng = np.random.default_rng(len(algo) + len(keys))
    tbl = _table(rng, 12_000, 30).append_column("rid", pa.array(np.arange(12_000)))
    if not keys:
        tbl = tbl.slice(0, 5000)
    cols = [f.median(col("v")).over().alias("med"), (col("v") - f.median(col("v")).over()).alias("dev"),
            f.percentile_disc(col("str"), 0.9).over().alias("p90"),
            f.percentile_cont(col("i"), 0.25).over().alias("q1"), f.sum(col("v")).over(running=True).alias("run"),
            f.row_number().alias("rn")]
    got = _run_map(tbl, cols, keys, presort, algo)
    rid = got.column("rid").to_pylist()
    med = Q.window_quantile(tbl, keys, "v", 0.5, Q.CONT)
    p90 = Q.window_quantile(tbl, keys, "str", 0.9, Q.DISC)
    q1 = Q.window_quantile(tbl, keys, "i", 0.25, Q.CONT)
    v = tbl.column("v").to_pylist()
    for j, r in enumerate(rid):
        assert _same(got.column("med")[j].as_py(), med[r], Q.CONT)
        assert _same(got.column("q1")[j].as_py(), q1[r], Q.CONT)
        assert got.column("p90")[j].as_py() == p90[r]
        d = None if v[r] is None or med[r] is None else v[r] - med[r]
        assert _same(got.column("dev")[j].as_py(), d, Q.CONT)
    if presort:  # the other window nodes, where the order inside a partition is unique
        exp = W.window_map(tbl, keys, OrderedDict([("rid", False)]),
                           [col("rid"), f.sum(col("v")).over(running=True).alias("run"), f.row_number().alias("rn")])
        for name in ["run", "rn"]:
            g = got.column(name).to_pylist()
            for j, r in enumerate(rid):
                a, b = g[j], exp[name][r]
                assert (a is None and b is None) or math.isclose(a, b, rel_tol=1e-9, abs_tol=1e-9), (name, r, a, b)
