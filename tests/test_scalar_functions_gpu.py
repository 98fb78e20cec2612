"""CASE, NULLIF, %, and the numeric functions on the device: every new K8 opcode against the numpy machine model
(tests/_func_sim.py) with every operand kind over edge values, the transcendental ones within the CUDA Programming
Guide's ulp bounds of the 50-digit reference (oracle/scalar.py), the host validation of malformed instructions, random
trees, and whole engine calls against the oracle."""
import math

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

import _func_sim as fsim
from fugue_b200 import _lib
from fugue_b200 import api as fa
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import SelectColumns, col, function, functions as ff
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import expressions as OX
from oracle import scalar as OS
from test_expr_compiler import _random, _same, _table
from test_scalar_functions_cpu import HAND, _num, _oracle, _run_f

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _edge_ints(n, rng):
    edge = np.array([I64_MIN, I64_MIN + 1, I64_MAX, -1, 0, 1, 7, -7, 2 ** 53 + 1, 2 ** 53 - 1, -(2 ** 53) - 1,
                     15, -15, 25, -25, 1049, -1050, 999_999_999_999_999_999], dtype=np.int64)
    return np.concatenate([edge, rng.integers(-10 ** 6, 10 ** 6, n - len(edge))])


def _edge_floats(n, rng):
    edge = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 5e-324, -5e-324, 2.2250738585072014e-308, 0.5,
                     -0.5, 1.5, 2.5, -2.5, 0.49999999999999994, 2.0 ** 53 + 1, 2.0 ** 53 - 1, 1e308, -1e308, 1.0,
                     -1.0, 3.0, 0.125, 1.005, 2.675, -8.0, 700.0, -745.0, 1e-10], dtype=np.float64)
    body = rng.standard_normal(n - len(edge)) * np.exp(rng.uniform(-20, 20, n - len(edge)))
    return np.concatenate([edge, body])


def _device(cols, valid):
    return ([torch.from_numpy(np.ascontiguousarray(c)).to(DEV) for c in cols],
            [None if v is None else torch.from_numpy(v).to(DEV) for v in valid])


UNARY = [K.X_ABS_I, K.X_ABS_F, K.X_FLOOR_F, K.X_CEIL_F, K.X_SQRT]
BINARY_I = [K.X_MOD_I, K.X_RMOD_I, K.X_GREATEST_I, K.X_LEAST_I]
BINARY_F = [K.X_MOD_F, K.X_RMOD_F, K.X_GREATEST_F, K.X_LEAST_F]


def _programs():
    """(name, program) pairs: acc loaded from column 0 (int) or 2 (float); operand B of every kind."""
    out = []
    for op in UNARY:
        src = 0 if op == K.X_ABS_I else 2
        out.append((f"un{op}", [(K.X_MOV, K.XK_COL, src, 0, 0), (op, K.XK_NONE, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)]))
        out.append((f"un{op}v", [(K.X_MOV, K.XK_COL, src + 1, 0, 0), (op, K.XK_NONE, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)]))
    for d in (-18, -3, -1):
        out.append((f"roundi{d}", [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_ROUND_I, K.XK_NONE, 0, 0, d & ((1 << 64) - 1)),
                                   (K.X_OUT, K.XK_NONE, 0, 0, 0)]))
    for d in (-18, -2, 0, 1, 2, 7, 18):
        out.append((f"roundf{d}", [(K.X_MOV, K.XK_COL, 2, 0, 0), (K.X_ROUND_F, K.XK_NONE, 0, 0, d & ((1 << 64) - 1)),
                                   (K.X_OUT, K.XK_NONE, 0, 0, 0)]))
    for ops, acc_col, other, imm, itof in ((BINARY_I, 0, 1, 7, False), (BINARY_F, 2, 3, fsim.sim._fb(2.5).item(), True)):
        for op in ops:
            kinds = [(K.XK_COL, other, 0, 0), (K.XK_COL, 4, 0, 0), (K.XK_IMM, 0, 0, imm), (K.XK_NULL, 0, 0, 0),
                     ("reg", other, 0, 0)]
            if itof:
                kinds.append((K.XK_COL, 1, K.XF_B_I2F, 0))  # an int column converted on load
            for kind, b, fl, im in kinds:
                if kind == "reg":
                    prog = [(K.X_MOV, K.XK_COL, b, 0, 0), (K.X_ST, K.XK_NONE, 2, 0, 0), (K.X_MOV, K.XK_COL, acc_col, 0, 0),
                            (op, K.XK_REG, 2, 0, 0)]
                else:
                    prog = [(K.X_MOV, K.XK_COL, acc_col, 0, 0), (op, kind, b, fl, im)]
                out.append((f"bin{op}k{kind}b{b}", prog + [(K.X_OUT, K.XK_NONE, 0, 0, 0)]))
    # SEL: condition from a bool column with NULLs in temporary 3, B of every kind
    cond = [(K.X_MOV, K.XK_COL, 5, 0, 0), (K.X_ST, K.XK_NONE, 3, 0, 0)]
    for kind, b, im in ((K.XK_COL, 3, 0), (K.XK_COL, 1, 0), (K.XK_IMM, 0, 42), (K.XK_NULL, 0, 0), (K.XK_REG, 1, 0)):
        pre = [(K.X_MOV, K.XK_COL, 3, 0, 0), (K.X_ST, K.XK_NONE, 1, 0, 0)] if kind == K.XK_REG else []
        out.append((f"sel{kind}b{b}", pre + cond + [(K.X_MOV, K.XK_COL, 2, 0, 0),
                                                    (K.X_SEL, kind, b, 3 << K.XF_COND_SHIFT, im),
                                                    (K.X_OUT, K.XK_NONE, 0, 0, 0)]))
    return out


@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 300_001])
def test_each_opcode_matches_the_model(n):
    rng = np.random.default_rng(n)
    m = max(n, 64)
    ints, floats = _edge_ints(m, rng)[:n], _edge_floats(m, rng)[:n]
    ints2 = rng.permutation(_edge_ints(m, rng))[:n]
    floats2 = rng.permutation(_edge_floats(m, rng))[:n]
    small = rng.integers(-3, 4, n).astype(np.int64)
    cond = rng.integers(0, 2, n).astype(np.uint8)
    cols = [ints, ints2, floats, floats2, small, cond]
    valid = [None, (rng.random(n) > 0.2).astype(np.uint8), None, (rng.random(n) > 0.2).astype(np.uint8),
             None, (rng.random(n) > 0.3).astype(np.uint8)]
    types = [K.T_I64, K.T_I64, K.T_F64, K.T_F64, K.T_I64, K.T_U8]
    dcols, dvalid = _device(cols, valid)
    for name, prog in _programs():
        out_t = K.T_F64 if any(op in (K.X_ABS_F, K.X_FLOOR_F, K.X_CEIL_F, K.X_SQRT, K.X_ROUND_F, K.X_SEL) + tuple(BINARY_F)
                               for op, *_ in prog) else K.T_I64
        dt = torch.float64 if out_t == K.T_F64 else torch.int64
        got, gv = K.eval_expr(n, DEV, dcols, dvalid, prog, [dt], [True], col_types=types, out_types=[out_t])
        want, wv = fsim.run(n, cols, valid, prog, [out_t], col_types=types)
        gv = gv[0].cpu().numpy()
        assert np.array_equal(gv, wv[0]), name
        g = got[0].cpu().numpy().view(np.uint64)[gv != 0]
        w = want[0].view(np.uint64)[wv[0] != 0]
        same = g == w
        if out_t == K.T_F64 and not any(op == K.X_ABS_F for op, *_ in prog):
            # which NaN a NaN operand gives back (its payload) is not specified for fmod; ABS keeps it
            same |= np.isnan(g.view(np.float64)) & np.isnan(w.view(np.float64))
        assert same.all(), name


def _ulps(a: float, b: float) -> int:
    ia = np.array([a]).view(np.int64)[0]
    ib = np.array([b]).view(np.int64)[0]
    ia = ia if ia >= 0 else -(ia & 0x7FFFFFFFFFFFFFFF)
    ib = ib if ib >= 0 else -(ib & 0x7FFFFFFFFFFFFFFF)
    return abs(int(ia) - int(ib))


def test_transcendental_within_ulp_bounds():
    rng = np.random.default_rng(7)
    n = 20_000
    x = _edge_floats(n, rng)
    x[-5000:] = rng.uniform(-700, 700, 5000)
    y = rng.permutation(_edge_floats(n, rng))
    y[-8000:] = np.round(rng.uniform(-6, 6, 8000), 1)
    y[:40] = [0.0, -0.0, 1.0, 2.0, 0.5, -1.0, 3.0, np.inf, -np.inf, np.nan] * 4
    dcols, dvalid = _device([x, y], [None, None])
    cases = [(K.X_EXP, OS.ref_exp, 1), (K.X_LN, OS.ref_ln, 1), (K.X_LOG10, OS.ref_log10, 1)]
    for op, ref, bound in cases + [(K.X_POW, OS.ref_pow, 2), (K.X_RPOW, None, 2)]:
        prog = [(K.X_MOV, K.XK_COL, 0, 0, 0), (op, K.XK_COL if op in (K.X_POW, K.X_RPOW) else K.XK_NONE, 1, 0, 0),
                (K.X_OUT, K.XK_NONE, 0, 0, 0)]
        got, gv = K.eval_expr(n, DEV, dcols, dvalid, prog, [torch.float64], [True], out_types=[K.T_F64])
        g, gv = got[0].cpu().numpy(), gv[0].cpu().numpy()
        for i in range(n):
            if op == K.X_POW:
                w = OS.ref_pow(float(x[i]), float(y[i]))
            elif op == K.X_RPOW:
                w = OS.ref_pow(float(y[i]), float(x[i]))
            else:
                w = ref(float(x[i]))
            if w is None:
                assert gv[i] == 0, (op, x[i], y[i])
                continue
            assert gv[i] == 1, (op, x[i], y[i])
            if math.isnan(w) or math.isinf(w) or w == 0:
                assert (math.isnan(w) and math.isnan(g[i])) or g[i] == w, (op, x[i], y[i], g[i], w)
            else:
                assert _ulps(float(g[i]), w) <= bound, (op, x[i], y[i], g[i], w)


def test_host_validation_rejects_malformed_instructions():
    n = 100
    c = [torch.zeros(n, dtype=torch.float64, device=DEV)]
    bad = [
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_SEL, K.XK_COL, 0, 4 << K.XF_COND_SHIFT, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_SEL, K.XK_NONE, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_MOD_F, K.XK_NONE, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_POW, K.XK_REG, 4, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_SQRT, K.XK_COL, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_ROUND_F, K.XK_NONE, 0, 0, 19), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_ROUND_I, K.XK_NONE, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_GREATEST_F, K.XK_COL, 0, 2, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
        [(K.X_MOV, K.XK_COL, 0, 0, 0), (K.X_LEAST_F + 1, K.XK_COL, 0, 0, 0), (K.X_OUT, K.XK_NONE, 0, 0, 0)],
    ]
    for prog in bad:  # refused by the host checks, before any launch
        with pytest.raises(_lib.FugueB200KernelError):
            K.eval_expr(n, DEV, c, [None], prog, [torch.float64], [False])
    torch.cuda.synchronize()


def _device_table(pdf):
    t = _table(pdf)
    return B200Table(t.schema, [c.to(DEV) for c in t.columns], [None if v is None else v.to(DEV) for v in t.valid])


def test_hand_picked_and_random_trees_on_the_device():
    pdf = _random(n=5000, seed=21)
    t = _device_table(pdf)
    named = [e.alias(f"c{i}") for i, e in enumerate(HAND)]
    want = _oracle(pdf, named)
    got = X.project(t, named)
    for e in named:
        _same(pd.Series(got.to_arrow().column(e.output_name).to_pandas()).convert_dtypes(), want[e.output_name], str(e))
    rng = np.random.default_rng(77)
    host = _table(pdf)
    checked = 0
    while checked < 150:
        e = _num(rng, int(rng.integers(1, 5))).alias("r")
        try:
            model, prog = _run_f(host, [e])
        except X._OutOfResources:
            continue
        if prog.cols == []:
            continue
        dev = X.project(t, [e]).to_arrow().column("r").to_pandas()
        _same(pd.Series(dev).convert_dtypes(), model[0], str(e))
        _same(model[0], _oracle(pdf, [e])["r"], str(e))
        checked += 1


def _frame(n=20_000, seed=3):
    rng = np.random.default_rng(seed)
    v = rng.integers(-1000, 1000, n)
    x = rng.standard_normal(n) * 100
    return pd.DataFrame({"k": rng.integers(0, 50, n), "v": v, "x": x, "w": rng.integers(-5, 6, n)})


def _rows(df):
    return sorted(tuple(None if (x is None or x is pd.NA or (isinstance(x, float) and math.isnan(x))) else x
                        for x in r) for r in df.itertuples(index=False))


def test_engine_select_filter_assign(engine):
    pdf = _frame()
    cols = [col("k"), ff.case([(col("v") > 0, col("x"))], -col("x")).alias("c"), (col("v") % 7).alias("m"),
            ff.nullif(col("w"), 0).alias("n"), ff.round(col("x"), 2).alias("r"), ff.sqrt(col("x")).alias("s"),
            ff.greatest(col("v"), col("w") * 100).alias("g"), function("ROUND", col("x"), -1).alias("r2"),
            function("abs", col("v")).alias("a")]
    got = fa.select(pdf, *cols, engine=engine, as_fugue=True).as_pandas()
    df, low, _ = OS.lower(pdf, cols)
    want = OX.select(df, SelectColumns(*low))
    assert _rows(got) == _rows(want)
    cond = (col("v") % 3 == 0) & (ff.abs(col("x")) > 50)
    got = fa.filter(pdf, cond, engine=engine, as_fugue=True).as_pandas()
    df, low, added = OS.lower(pdf, [cond])
    assert _rows(got) == _rows(OX.filter_rows(df, low[0]).drop(columns=added))
    got = fa.assign(pdf, q=ff.floor(col("x")), engine=engine, as_fugue=True).as_pandas()
    assert np.array_equal(got["q"].to_numpy(), np.floor(pdf["x"].to_numpy()))


def test_engine_aggregate_group_by_string_case_and_having(engine):
    pdf = _frame()
    got = fa.aggregate(pdf, "k", engine=engine, as_fugue=True,
                       s=ff.sum(ff.case([(col("v") > 0, col("v"))], 0)),
                       c=ff.count(ff.case([(col("x") > 0, 1)])), a=ff.avg(ff.abs(col("x")))).as_pandas()
    g = pdf.groupby("k")
    want = pd.DataFrame({"k": sorted(pdf["k"].unique())})
    want["s"] = want["k"].map(g.apply(lambda d: d["v"].clip(lower=0).sum()))
    want["c"] = want["k"].map(g.apply(lambda d: int((d["x"] > 0).sum())))
    got = got.sort_values("k").reset_index(drop=True)
    assert got["s"].tolist() == want["s"].tolist() and got["c"].tolist() == want["c"].tolist()
    a = want["k"].map(g.apply(lambda d: d["x"].abs().mean()))
    assert np.allclose(got["a"].to_numpy(), a.to_numpy(), rtol=1e-12)
    grade = ff.case([(col("v") >= 500, "A"), (col("v") >= 0, "B")], "C").alias("grade")
    got = fa.select(pdf, grade, ff.count(col("v")).alias("n"), engine=engine, as_fugue=True).as_pandas()
    lab = np.where(pdf["v"] >= 500, "A", np.where(pdf["v"] >= 0, "B", "C"))
    assert dict(zip(got["grade"], got["n"])) == dict(zip(*np.unique(lab, return_counts=True)))
    got = fa.select(pdf, col("k"), ff.sum(col("v")).alias("s"), having=ff.sum(col("v")) % 2 == 0, engine=engine,
                    as_fugue=True).as_pandas()
    sums = pdf.groupby("k")["v"].sum()
    assert sorted(got["k"].tolist()) == sorted(sums[sums % 2 == 0].index.tolist())


def test_raw_sql_with_every_keyword(engine):
    pdf = _frame(n=5000)
    got = fa.raw_sql("SELECT k, CASE WHEN v > 0 THEN 'pos' WHEN v < 0 THEN 'neg' ELSE 'zero' END AS sgn, "
                     "CASE w WHEN 1 THEN 10 WHEN 2 THEN 20 END AS cw, IF(v > 0, 1, 0) AS i1, IIF(v < 0, 1.5, 2.5) AS i2, "
                     "NULLIF(w, 0) AS nz, IFNULL(NULLIF(w, 0), -1) AS fz, v % 7 AS m1, MOD(v, 5) AS m2, ABS(v) AS av, "
                     "FLOOR(x) AS fl, CEIL(x) AS ce, CEILING(x) AS ce2, ROUND(x, 1) AS ro, SQRT(ABS(x)) AS sq, "
                     "EXP(x / 100) AS ex, LN(ABS(x) + 1) AS lnx, LOG10(ABS(x) + 1) AS lg, POWER(x, 2) AS p2, "
                     "POW(2, w) AS p3, GREATEST(v, w, 0) AS gr, LEAST(x, 0.5) AS le FROM", pdf,
                     "WHERE v % 2 = 0", engine=engine, as_fugue=True).as_pandas()
    sub = pdf[pdf["v"] % 2 == 0].reset_index(drop=True)
    assert len(got) == len(sub)
    got = got.reset_index(drop=True)
    assert got["sgn"].tolist() == np.where(sub["v"] > 0, "pos", np.where(sub["v"] < 0, "neg", "zero")).tolist()
    assert got["m1"].tolist() == [OS.mod(int(v), 7, False) for v in sub["v"]]
    assert got["fz"].tolist() == [w if w != 0 else -1 for w in sub["w"]]
    assert got["gr"].tolist() == [max(v, w, 0) for v, w in zip(sub["v"], sub["w"])]
    p2 = sub["x"].to_numpy() ** 2
    assert all(_ulps(float(a), float(b)) <= 2 for a, b in zip(got["p2"].to_numpy(), p2))  # CUDA pow: 2 ulp
    assert np.array_equal(got["sq"].to_numpy(), np.sqrt(np.abs(sub["x"].to_numpy())))


def test_window_map_with_case_and_round(engine):
    pdf = _frame(n=4000)
    pdf["rid"] = np.arange(len(pdf))
    cm = ColumnMap("rid", ff.sum(ff.case([(col("v") > 0, col("v"))], 0)).over(running=True).alias("rs"),
                   ff.round(ff.avg(col("x")).over(), 2).alias("ra"))
    got = fa.transform(pdf, cm, schema="rid:long,rs:long,ra:double", partition=PartitionSpec(by="k", presort="rid"),
                       engine=engine, as_fugue=True).as_pandas().sort_values("rid").reset_index(drop=True)
    want_rs = pdf.assign(pv=pdf["v"].clip(lower=0)).groupby("k")["pv"].cumsum()
    assert got["rs"].tolist() == want_rs.tolist()
    means = pdf.groupby("k")["x"].transform("mean")
    assert np.allclose(got["ra"].to_numpy(), [OS.round_(float(m), 2, True) for m in means], rtol=0, atol=1e-2 + 1e-12)


def test_column_map_with_mod_is_not_fused(engine):
    pdf = _frame(n=50_000)
    t = B200Table.from_arrow(pa.Table.from_pandas(pdf, preserve_index=False), DEV)
    cm = ColumnMap("k", (col("v") % 7).alias("m"))
    assert cm.fusion_units(t) is None  # partition, then the evaluator
    assert ColumnMap("k", (col("v") * 7).alias("m")).fusion_units(t) is not None
    got = fa.transform(pdf, cm, schema="k:long,m:long", partition=PartitionSpec(by="k", algo="hash", num=16),
                       engine=engine, as_fugue=True).as_pandas()
    assert sorted(zip(got["k"], got["m"])) == sorted(zip(pdf["k"], [OS.mod(int(v), 7, False) for v in pdf["v"]]))
