"""Date and timestamp expressions on the device: every temporal opcode bit for bit against the numpy machine model,
random values against the oracle, host validation, and the engine routes (select / filter / assign / aggregate / SQL /
window maps) against the oracle."""
import datetime as dt

import numpy as np
import pyarrow as pa
import pytest
import torch

import _temporal_sim as tsim
from fugue_b200 import _lib
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import col, functions as f, lit
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import temporal as OT
from test_temporal_cpu import CODE, I64_MAX, I64_MIN, UNITS, edge_values

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
OUT = (K.X_OUT, K.XK_NONE, 0, 0, 0)


@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _device(cols, valid):
    return ([torch.from_numpy(np.ascontiguousarray(c)).to(DEV) for c in cols],
            [None if v is None else torch.from_numpy(v).to(DEV) for v in valid])


def _check(n, cols, valid, prog, name):
    dcols, dvalid = _device(cols, valid)
    got, gv = K.eval_expr(n, DEV, dcols, dvalid, prog, [torch.int64], [True])
    want, wv = tsim.run(n, cols, valid, prog, [K.T_I64])
    gv = gv[0].cpu().numpy()
    assert np.array_equal(gv, wv[0]), name
    assert np.array_equal(got[0].cpu().numpy()[gv != 0], want[0][wv[0] != 0]), name


def _values(unit, n, rng):
    edge = np.array(edge_values(unit), dtype=np.int64)
    span = 2 ** 31 - 1 if unit == "D" else 2 ** 63 - 1
    body = rng.integers(-span, span, max(n, len(edge)) - len(edge) + 1)
    return np.concatenate([edge, body])[:n]


@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 300_001])
def test_each_temporal_opcode_matches_the_model(n):
    rng = np.random.default_rng(n)
    months = rng.choice(np.array([0, 1, -1, 12, -12, 13, -13, 4800, -4800, I64_MAX, I64_MIN], dtype=np.int64), n)
    mvalid = (rng.random(n) > 0.2).astype(np.uint8)
    for unit, code in CODE.items():
        x = rng.permutation(_values(unit, n, rng))
        cols, valid = [x, months, months], [(rng.random(n) > 0.2).astype(np.uint8), None, mvalid]
        mov = (K.X_MOV, K.XK_COL, 0, 0, 0)
        for op, words in ((K.X_TS_PART, K.TIME_FIELDS), (K.X_TS_TRUNC, K.TIME_PARTS), (K.X_TS_INDEX, K.TIME_PARTS)):
            for w in range(len(words)):
                _check(n, cols, valid, [mov, (op, K.XK_NONE, 0, 0, w | code << 8), OUT], (unit, op, words[w]))
        fl = code << K.XF_UNIT_SHIFT
        for name, ins in (("col", (K.X_TS_ADDMON, K.XK_COL, 1, fl, 0)), ("nullable", (K.X_TS_ADDMON, K.XK_COL, 2, fl, 0)),
                          ("imm", (K.X_TS_ADDMON, K.XK_IMM, 0, fl, -13 & ((1 << 64) - 1))),
                          ("null", (K.X_TS_ADDMON, K.XK_NULL, 0, fl, 0))):
            _check(n, cols, valid, [mov, ins, OUT], (unit, "addmon", name))
        _check(n, cols, valid, [(K.X_MOV, K.XK_COL, 1, 0, 0), (K.X_ST, K.XK_NONE, 2, 0, 0), mov,
                                (K.X_TS_ADDMON, K.XK_REG, 2, fl, 0), OUT], (unit, "addmon", "reg"))
    x = rng.permutation(_values("ns", n, rng))
    for b in (1, 1000, 86400, 86_400_000_000_000):
        for op in (K.X_MULSAT_I, K.X_FLOORDIV_I):
            _check(n, [x], [(rng.random(n) > 0.2).astype(np.uint8)], [(K.X_MOV, K.XK_COL, 0, 0, 0), (op, K.XK_IMM, 0, 0, b), OUT],
                   (op, b))


@pytest.mark.parametrize("unit", list(UNITS))
def test_a_million_random_values_match_the_oracle(unit):
    rng = np.random.default_rng(17)
    n = 1_000_000
    span = 2 ** 31 - 1 if unit == "D" else min(2 ** 63 - 1, (2 ** 31 - 1) * OT.PER_DAY[unit])
    x = rng.integers(-span, span, n)
    dcols, dvalid = _device([x], [None])
    check = rng.integers(0, n, 4000)  # the oracle is one Python value at a time: a sample of the rows
    code = CODE[unit]
    for op, words, fn in ((K.X_TS_PART, K.TIME_FIELDS, OT.extract), (K.X_TS_TRUNC, K.TIME_PARTS, OT.date_trunc)):
        for w, word in enumerate(words):
            prog = [(K.X_MOV, K.XK_COL, 0, 0, 0), (op, K.XK_NONE, 0, 0, w | code << 8), OUT]
            got = K.eval_expr(n, DEV, dcols, dvalid, prog, [torch.int64], [False])[0][0].cpu().numpy()
            assert np.array_equal(got, tsim.run(n, [x], [None], prog, [K.T_I64])[0][0]), (unit, word)
            assert [int(got[i]) for i in check] == [fn(word, int(x[i]), unit) for i in check], (unit, word)
    prog = [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_TS_ADDMON, K.XK_IMM, 0, code << K.XF_UNIT_SHIFT, 25), OUT]
    got = K.eval_expr(n, DEV, dcols, dvalid, prog, [torch.int64], [False])[0][0].cpu().numpy()
    assert [int(got[i]) for i in check] == [OT.add_months(int(x[i]), 25, unit) for i in check]


def test_host_validation_rejects_malformed_temporal_instructions():
    n = 100
    c = [torch.zeros(n, dtype=torch.int64, device=DEV)]
    mov = (K.X_MOV, K.XK_COL, 0, 0, 0)
    bad = [(K.X_MULSAT_I, K.XK_IMM, 0, 0, 0), (K.X_MULSAT_I, K.XK_COL, 0, 0, 0), (K.X_FLOORDIV_I, K.XK_IMM, 0, 0, 0),
           (K.X_FLOORDIV_I, K.XK_IMM, 0, 0, -5 & ((1 << 64) - 1)), (K.X_FLOORDIV_I, K.XK_NONE, 0, 0, 7),
           (K.X_TS_PART, K.XK_NONE, 0, 0, len(K.TIME_FIELDS)), (K.X_TS_PART, K.XK_NONE, 0, 0, 5 << 8),
           (K.X_TS_PART, K.XK_COL, 0, 0, 0), (K.X_TS_TRUNC, K.XK_NONE, 0, 0, len(K.TIME_PARTS)),
           (K.X_TS_INDEX, K.XK_NONE, 0, 0, -1 & ((1 << 64) - 1)), (K.X_TS_INDEX, K.XK_IMM, 0, 0, 0),
           (K.X_TS_ADDMON, K.XK_NONE, 0, 0, 0), (K.X_TS_ADDMON, K.XK_IMM, 0, 5 << K.XF_UNIT_SHIFT, 1),
           (K.X_TS_ADDMON, K.XK_IMM, 0, K.XF_B_I2F, 1), (K.X_TS_ADDMON + 1, K.XK_COL, 0, 0, 0),
           (K.X_TS_ADDMON + 1, K.XK_NONE, 0, 0, 0)]
    for ins in bad:  # refused by the host checks, before any launch
        with pytest.raises(_lib.FugueB200KernelError):
            K.eval_expr(n, DEV, c, [None], [mov, ins, OUT], [torch.int64], [False])
    torch.cuda.synchronize()


# ---- engine routes -------------------------------------------------------------------------------------------
def _frame(tp, n=20_000, seed=3):
    """An arrow table with a temporal column ``t`` (NULLs), an earlier one ``t0``, a key and a value; and the same
    rows as storage integers for the oracle."""
    rng = np.random.default_rng(seed)
    per = OT.PER_DAY[OT.unit_of(tp)]
    base = OT.days_of(2023, 6, 1) * per
    t = base + rng.integers(0, 500 * per, n)
    t0 = t - rng.integers(0, 90 * per, n)
    tv = [None if rng.random() < 0.1 else int(v) for v in t]
    ints = {"t": tv, "t0": [int(v) for v in t0], "key": [int(v) for v in rng.integers(0, 20, n)],
            "v": [int(v) for v in rng.integers(-1000, 1000, n)], "rid": list(range(n))}
    raw = pa.int32() if pa.types.is_date32(tp) else pa.int64()
    tbl = pa.table({"t": pa.array(tv, raw).cast(tp), "t0": pa.array(ints["t0"], raw).cast(tp),
                    "key": pa.array(ints["key"], pa.int64()), "v": pa.array(ints["v"], pa.int64()),
                    "rid": pa.array(ints["rid"], pa.int64())})
    return tbl, ints


def _ints(tbl, names):
    """Rows of an arrow result with temporal columns as their storage integers."""
    cols = []
    for nm in names:
        c = tbl.column(nm)
        if OT.unit_of(c.type):
            c = c.cast(pa.int32() if pa.types.is_date32(c.type) else pa.int64())
        cols.append(c.to_pylist())
    return sorted(zip(*cols), key=lambda r: tuple((x is None, x) for x in r))


def _srt(rows):
    return sorted(rows, key=lambda r: tuple((x is None, x) for x in r))


TYPES = [pa.date32(), pa.timestamp("us"), pa.timestamp("ns", tz="UTC")]


@pytest.mark.parametrize("tp", TYPES, ids=str)
def test_engine_select_filter_assign(engine, tp):
    tbl, ints = _frame(tp)
    u = OT.unit_of(tp)
    got = fa.select(tbl, col("rid"), f.year(col("t")).alias("y"), f.extract("week", col("t")).alias("w"),
                    f.date_trunc("month", col("t")).alias("m"), f.add_months(col("t"), col("key") - 10).alias("a"),
                    f.datediff("day", col("t0"), col("t")).alias("dd"), f.extract("epoch", col("t")).alias("ep"),
                    engine=engine, as_fugue=True).as_arrow()
    assert got.schema.field("m").type == tp and got.schema.field("a").type == tp
    assert got.schema.field("y").type == pa.int64() and got.schema.field("ep").type == pa.float64()
    want = [(r, OT.extract("year", t, u), OT.extract("week", t, u), OT.date_trunc("month", t, u), OT.add_months(t, k - 10, u),
             OT.datediff("day", t0, u, t, u), OT.extract("epoch", t, u))
            for r, t, t0, k in zip(ints["rid"], ints["t"], ints["t0"], ints["key"])]
    assert _ints(got, ["rid", "y", "w", "m", "a", "dd", "ep"]) == _srt(want)
    cut = dt.datetime(2024, 6, 1)
    got = fa.filter(tbl, col("t") < lit(cut), engine=engine, as_fugue=True).as_arrow()
    keep = [r for r, t in zip(ints["rid"], ints["t"]) if t is not None and OT.compare("<", t, u, cut)]
    assert sorted(got.column("rid").to_pylist()) == keep and 0 < len(keep) < len(ints["rid"])
    got = fa.assign(tbl, due=f.add_months(col("t"), 1), age=f.datediff("day", col("t0"), col("t")), engine=engine,
                    as_fugue=True).as_arrow()
    assert got.schema.field("due").type == tp
    want = [(r, OT.add_months(t, 1, u), OT.datediff("day", t0, u, t, u)) for r, t, t0 in zip(ints["rid"], ints["t"], ints["t0"])]
    assert _ints(got, ["rid", "due", "age"]) == _srt(want)


@pytest.mark.parametrize("tp", TYPES, ids=str)
def test_engine_aggregate_having_and_raw_sql(engine, tp):
    tbl, ints = _frame(tp)
    u = OT.unit_of(tp)
    got = fa.raw_sql("SELECT DATE_TRUNC('month', t) AS m, key, SUM(v) AS s FROM", tbl,
                     "WHERE t >= DATE '2024-01-01' AND EXTRACT(dow FROM t) NOT IN (0, 6) "
                     "GROUP BY DATE_TRUNC('month', t), key ORDER BY m", engine=engine, as_fugue=True).as_arrow()
    assert got.schema.field("m").type == tp
    sums = {}
    for t, k, v in zip(ints["t"], ints["key"], ints["v"]):
        if t is not None and OT.compare(">=", t, u, dt.date(2024, 1, 1)) and OT.extract("dow", t, u) not in (0, 6):
            g = (OT.date_trunc("month", t, u), k)
            sums[g] = sums.get(g, 0) + v
    assert _ints(got, ["m", "key", "s"]) == _srt([(m, k, s) for (m, k), s in sums.items()])
    ms = got.column("m").cast(pa.int32() if u == "D" else pa.int64()).to_pylist()
    assert ms == sorted(ms)  # ORDER BY the aliased expression
    got = fa.select(tbl, f.year(col("t")).alias("y"), col("key"), f.sum(col("v")).alias("s"),
                    f.max(f.extract("doy", col("t"))).alias("mx"), having=f.sum(col("v")) > 0, engine=engine,
                    as_fugue=True).as_arrow()
    acc = {}
    for t, k, v in zip(ints["t"], ints["key"], ints["v"]):
        g = (None if t is None else OT.extract("year", t, u), k)
        s, mx = acc.get(g, (0, None))
        d = None if t is None else OT.extract("doy", t, u)
        acc[g] = (s + v, mx if d is None else d if mx is None else max(mx, d))
    assert _ints(got, ["y", "key", "s", "mx"]) == _srt([(y, k, s, mx) for (y, k), (s, mx) in acc.items() if s > 0])


@pytest.mark.parametrize("tp", TYPES, ids=str)
def test_window_map_arguments_and_outputs(engine, tp):
    tbl, ints = _frame(tp, n=4000)
    tbl = tbl.filter(pa.compute.is_valid(tbl.column("t")))
    u = OT.unit_of(tp)
    cm = ColumnMap("rid", (col("t") - f.lag(col("t"))).alias("gap"), f.max(f.year(col("t"))).over().alias("my"),
                   f.date_trunc("week", col("t")).cast("long").alias("wk"))
    t = B200Table.from_arrow(tbl, DEV)
    assert ColumnMap("key", f.date_trunc("week", col("t")).alias("wk")).fusion_units(t) is None  # never in the scatter
    got = fa.transform(tbl, cm, schema="rid:long,gap:long,my:long,wk:long", partition=PartitionSpec(by="key", presort="rid"),
                       engine=engine, as_fugue=True).as_arrow()
    rows = [(r, t_, k) for r, t_, k in zip(ints["rid"], ints["t"], ints["key"]) if t_ is not None]
    want, last, top = [], {}, {}
    for r, t_, k in rows:
        top[k] = max(top.get(k, -10 ** 9), OT.extract("year", t_, u))
    for r, t_, k in rows:
        want.append((r, None if k not in last else t_ - last[k], top[k], OT.date_trunc("week", t_, u)))
        last[k] = t_
    assert _ints(got, ["rid", "gap", "my", "wk"]) == _srt(want)


def test_other_time_zones_raise_before_any_launch(engine, monkeypatch):
    tbl, _ = _frame(pa.timestamp("us"), n=100)
    tbl = tbl.set_column(0, "t", tbl.column("t").cast(pa.timestamp("us", tz="Europe/Paris")))
    calls = []
    real = K.eval_expr
    monkeypatch.setattr(K, "eval_expr", lambda *a, **k: calls.append(1) or real(*a, **k))
    for fn in (lambda: fa.select(tbl, f.year(col("t")).alias("y"), engine=engine),
               lambda: fa.filter(tbl, f.date_trunc("day", col("t")) > lit(dt.date(2024, 1, 1)), engine=engine)):
        with pytest.raises(NotImplementedError):
            fn()
    assert calls == []
    got = fa.filter(tbl, col("t") >= lit(dt.datetime(2024, 1, 1)), engine=engine, as_fugue=True).as_arrow()  # the UTC instant
    assert calls and 0 < got.num_rows < 100
