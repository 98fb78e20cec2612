"""Host-side expression compiler (fugue_b200/expr.py) checked WITHOUT a GPU: programs are generated for
a table of CPU tensors, executed by the numpy model of the accumulator machine (tests/_expr_sim.py)
and compared with oracle/expressions.py.  The -m gpu tests run the same programs on the device."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200.column import SelectColumns, col, functions as ff, lit, null
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table, _storage_dtype, expr_type, narrow, widen
from oracle import expressions as OX
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _expr_sim as sim  # noqa: E402


def _table(pdf: pd.DataFrame) -> B200Table:
    fields, cols, valids = [], [], []
    for name in pdf.columns:
        s = pdf[name]
        na = s.isna().to_numpy()
        if pd.api.types.is_bool_dtype(s.dtype):
            tp, arr = pa.bool_(), s.fillna(False).to_numpy(dtype=np.uint8)
        elif pd.api.types.is_float_dtype(s.dtype):
            tp, arr = pa.float64(), np.nan_to_num(s.to_numpy(dtype=np.float64, na_value=0.0))
        else:
            bits = 32 if str(s.dtype).lower() == "int32" else 64
            tp = pa.int32() if bits == 32 else pa.int64()
            arr = s.fillna(0).to_numpy(dtype=np.int32 if bits == 32 else np.int64)
        fields.append(pa.field(name, tp))
        cols.append(torch.from_numpy(np.ascontiguousarray(arr)))
        valids.append(torch.from_numpy((~na).astype(np.uint8)) if na.any() else None)
    return B200Table(Schema(fields), cols, valids)


def _run(t: B200Table, exprs):
    """Compile every expression into ONE program and simulate it; returns pandas nullable columns."""
    prog = X._Program(t)
    meta = []
    for e in exprs:
        cls, nullable = prog.compile(e, top=True)
        dtype = {"i": torch.int64, "f": torch.float64, "b": torch.uint8}[cls]
        prog.output(dtype, True)
        meta.append(cls)
    cols = [t.columns[i].numpy() for i in prog.cols]
    valid = [None if t.valid[i] is None else t.valid[i].numpy() for i in prog.cols]
    outs, outv = sim.run(t.num_rows, cols, valid, prog.ins, [o[2] for o in prog.outs],
                         col_types=[expr_type(t.schema.types[i]) for i in prog.cols])
    res = []
    for cls, o, v in zip(meta, outs, outv):
        dt = {"i": "Int64", "f": "Float64", "b": "boolean"}[cls]
        arr = pd.array(o.astype(bool) if cls == "b" else o, dtype=dt)
        arr[v == 0] = pd.NA
        res.append(pd.Series(arr))
    return res, prog


def _random(n=4000, seed=3):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n)
    x[rng.random(n) < 0.2] = np.nan
    return pd.DataFrame({
        "a": rng.integers(-50, 50, n).astype(np.int64), "b": rng.integers(0, 7, n).astype(np.int32), "x": x,
        "y": rng.standard_normal(n) * 10,
        "g": pd.array(np.where(rng.random(n) < 0.1, None, rng.integers(0, 20, n)), dtype="Int64"),
        "p": pd.array(np.where(rng.random(n) < 0.15, None, rng.random(n) < 0.5), dtype="boolean")})


def _same(got: pd.Series, want: pd.Series, name: str):
    gn, wn = got.isna().to_numpy(), want.isna().to_numpy()
    assert (gn == wn).all(), name
    g = got[~gn].to_numpy(dtype=np.float64)
    w = want[~wn].to_numpy(dtype=np.float64)
    assert np.array_equal(g, w, equal_nan=True), name


EXPRS = [
    col("a") * col("b") - 3, col("x") / col("y"), col("a") / col("b"), -col("x"), -col("b"), 10 - col("a"),
    2.5 / col("y"), (col("a") + col("b")) * (col("x") - col("y")), (col("a") - 1) / (col("b") + 1),
    (col("x") > 0) & col("p"), (col("x") > 0) | col("p"), ~col("p"), col("x").is_null() | (col("a") >= col("b")),
    col("g") == col("b"), col("g") != 3, 3 < col("g"), (col("a") > 0) & ((col("b") < 3) | (col("x") > col("y"))),
    col("p") & null(), col("p") | null(), null() & col("p"), lit(True) & col("p"), col("a") + null(),
    ff.coalesce(col("x"), col("y")), ff.coalesce(col("g"), -1), ff.coalesce(col("g"), col("x"), 0.5),
    ff.coalesce(col("x") * 2, col("g") + 1, col("a")), ff.coalesce(null(), col("g")),
    (col("a") + 1.5).cast(int), col("x").cast("long"), col("b").cast(float), (col("a") > 0).cast(int),
    col("g").cast(bool), (col("x") * 3).cast(bool) & col("p"), (col("a") & col("b")), ~(col("a") - 1),
    (col("x") + col("y") > 0) | (col("g").is_null() & col("p")), (col("x").not_null() & (col("x") < 0.5)),
]


def test_compiled_programs_match_oracle():
    pdf = _random()
    t = _table(pdf)
    named = [e.alias(f"c{i}") for i, e in enumerate(EXPRS)]
    want = OX.select(pdf, SelectColumns(*named))
    for lo in range(0, len(named), 8):  # several expressions share one program
        got, prog = _run(t, named[lo:lo + 8])
        assert len(prog.ins) <= K.EXPR_MAX_INS
        for e, s in zip(named[lo:lo + 8], got):
            _same(s, want[e.output_name], str(e))


def test_leaf_operands_need_no_temporaries():
    t = _table(_random(64))
    prog = X._Program(t)
    prog.compile(col("x") * col("y") + col("a"))
    assert [i[0] for i in prog.ins] == [K.X_MOV, K.X_MUL_F, K.X_ADD_F]
    assert prog.ins[2][3] == K.XF_B_I2F and all(i[1] == K.XK_COL for i in prog.ins)
    prog = X._Program(t)
    prog.compile((col("x") > 0) & (col("y") < 0.5))
    assert [i[0] for i in prog.ins] == [K.X_MOV, K.X_GT_F, K.X_ST, K.X_MOV, K.X_LT_F, K.X_AND]
    assert len(prog.free) == K.EXPR_NREGS
    prog = X._Program(t)
    prog.compile(10 - col("a") * 2)
    assert [i[0] for i in prog.ins] == [K.X_MOV, K.X_MUL_I, K.X_RSUB_I]
    prog = X._Program(t)
    prog.compile(col("a") / col("b"))       # integer leaves are converted while they are loaded
    assert [(i[0], i[3]) for i in prog.ins] == [(K.X_MOV, K.XF_B_I2F), (K.X_DIV_F, K.XF_B_I2F)]
    prog = X._Program(t)
    prog.compile((col("a") + 1) / 2)        # ... but not after integer arithmetic
    assert [i[0] for i in prog.ins] == [K.X_MOV, K.X_ADD_I, K.X_I2F, K.X_DIV_F]


def test_resource_limits_and_errors():
    t = _table(_random(64))
    deep = col("a")
    for i in range(6):  # right-nested compound operands: one temporary per level
        deep = (col("a") + i) * (deep - col("b") * 2)
    with pytest.raises(X._OutOfResources):
        X._Program(t).compile(deep)
    with pytest.raises(KeyError):
        X._Program(t).compile(col("nope") + 1)
    with pytest.raises(ValueError):
        X._Program(t).compile(ff.max(col("a")) + 1)
    with pytest.raises(NotImplementedError):
        X._Program(t).compile(col("a") + "s")


def _typed_table():
    """uint16 / uint32 / float16 columns in their storage tensors (int16 / int32 / int16), with the frame of
    their values."""
    u16 = np.array([0, 1, 32767, 32768, 40000, 65535], dtype=np.uint16)
    u32 = np.array([1, 2 ** 31 - 1, 2 ** 31, 3_000_000_000, 2 ** 32 - 1, 7], dtype=np.uint32)
    h = np.array([1.5, -2.0, 0.25, -0.0, 65504, 6e-8], dtype=np.float16)
    t = B200Table(Schema([pa.field("w", pa.uint16()), pa.field("u", pa.uint32()), pa.field("h", pa.float16())]),
                  [torch.from_numpy(a.view(s).copy()) for a, s in ((u16, np.int16), (u32, np.int32), (h, np.int16))],
                  [None, torch.from_numpy(np.array([1, 1, 1, 0, 1, 1], dtype=np.uint8)), None])
    pdf = pd.DataFrame({"w": pd.array(u16.astype(np.int64), dtype="Int64"),
                        "u": pd.array([int(v) if ok else None for v, ok in zip(u32.tolist(), [1, 1, 1, 0, 1, 1])],
                                      dtype="Int64"),
                        "h": pd.array(h.astype(np.float64), dtype="Float64")})
    return t, pdf


def test_unsigned_and_half_columns_are_read_by_value():
    t, pdf = _typed_table()
    exprs = [col("u") + 1, col("u") > 5, col("w") * 2 - col("u"), col("w") > 32767, col("h") * 2.0, col("h") < 0,
             col("h") + col("w"), col("u") / col("h"), (col("h") * 3).cast(int), ff.coalesce(col("u"), col("w"))]
    named = [e.alias(f"c{i}") for i, e in enumerate(exprs)]
    got, _ = _run(t, named)
    want = OX.select(pdf, SelectColumns(*named))
    for e, s in zip(named, got):
        _same(s, want[e.output_name], str(e))


def test_narrow_outputs_store_by_value():
    """A cast to uint16 / uint32 keeps the low bits; a cast to float16 rounds to nearest even once."""
    t, _ = _typed_table()
    x = pd.DataFrame({"x": [1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 65519.99, 65520.0, 2.0 ** -25, -3 * 2.0 ** -26]})
    tx = _table(x)
    for tab, e, tp, want in [
            (t, col("u") * 3, pa.uint32(), (np.array([1, 2 ** 31 - 1, 2 ** 31, 0, 2 ** 32 - 1, 7], np.int64) * 3
                                            ).astype(np.uint32)),
            (t, col("u") - 1, pa.uint16(), (np.array([1, 2 ** 31 - 1, 2 ** 31, 0, 2 ** 32 - 1, 7], np.int64) - 1
                                            ).astype(np.uint16)),
            (tx, col("x"), pa.float16(), x["x"].to_numpy().astype(np.float16))]:
        prog = X._Program(tab)
        prog.compile(e.cast(tp), top=True)
        prog.output(_storage_dtype(tp), False, expr_type(tp))
        cols = [tab.columns[i].numpy() for i in prog.cols]
        outs, outv = sim.run(tab.num_rows, cols,
                             [None if tab.valid[i] is None else tab.valid[i].numpy() for i in prog.cols], prog.ins,
                             [o[2] for o in prog.outs], col_types=[expr_type(tab.schema.types[i]) for i in prog.cols])
        ok = outv[0].astype(bool)
        got = outs[0].view(want.dtype)
        assert np.array_equal(got[ok], want[ok]) and (outs[0][~ok] == 0).all(), (e, got, want)
    assert np.array_equal(got, np.array([1.0, 1.001953125, 65504, np.inf, 0.0, -5.960464477539063e-08],
                                        dtype=np.float16))


def test_f2i_saturates_and_maps_nan_to_int64_min():
    """The model's FB_X_F2I is the device's: saturation at the int64 bounds, NaN -> INT64_MIN."""
    v = np.array([np.inf, -np.inf, np.nan, -np.nan, 1e300, -1e300, 2.0 ** 63, -2.0 ** 63, -2.5, 2.5, 2.0 ** 63 - 1024])
    t = B200Table(Schema([pa.field("x", pa.float64())]), [torch.from_numpy(v)], [None])
    prog = X._Program(t)
    prog.compile(col("x").cast(int), top=True)
    prog.output(torch.int64, False)
    outs, _ = sim.run(len(v), [v], [None], prog.ins, [K.T_I64])
    i64 = np.iinfo(np.int64)
    assert outs[0].tolist() == [i64.max, i64.min, i64.min, i64.min, i64.max, i64.min, i64.max, i64.min, -2, 2, 2 ** 63 - 1024]


def test_widen_reads_every_storage_type_by_value():
    cases = [(pa.uint16(), np.array([0, 40000, 65535], np.uint16), np.int16),
             (pa.uint32(), np.array([0, 2 ** 31, 2 ** 32 - 1], np.uint32), np.int32),
             (pa.float16(), np.array([-0.0, 65504, 6e-8], np.float16), np.int16),
             (pa.int8(), np.array([-128, 127, 0], np.int8), np.int8),
             (pa.float32(), np.array([1e-45, -3.5, np.inf], np.float32), np.float32)]
    for tp, v, st in cases:
        w = widen(torch.from_numpy(v.view(st).copy()), tp)
        want = v.astype(np.float64 if pa.types.is_floating(tp) else np.int64)
        assert np.array_equal(w.numpy(), want) and np.array_equal(np.signbit(w.numpy()), np.signbit(want)), tp
        back = narrow(w, tp).numpy()
        assert back.dtype == st and np.array_equal(back.view(np.uint8), v.view(np.uint8)), tp
