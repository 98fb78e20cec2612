"""The device expression evaluator (K8, ``fb_eval_expr``) against exact references, at the types, operands,
sizes and program shapes where it can go wrong.

* every opcode with every operand kind (a column with and without validity, an immediate, a temporary,
  NULL, an integer operand converted by ``XF_B_I2F``) over int and float edge values, checked against
  values computed here with Python ints and ``math`` and against the numpy model ``tests/_expr_sim.py``;
* every input storage type (uint16 / uint32 / float16 included) into every output type;
* sizes around the 2048-row tile and the grid-stride loop, with all four temporaries live;
* programs at the limits: 96 instructions, 16 columns, 16 outputs;
* the 600 seeded trees of ``test_expr_random.py`` and 300 more over a table of every storage type, on the
  device, against the model and ``oracle/expressions.py``;
* ``select`` / ``filter`` / ``assign``, ``aggregate`` and window aggregates of every numeric type, through
  the engine, against ``oracle/expressions.py``, pandas and ``oracle/window.py``.

Values and validity are compared bit for bit; a NULL row stores 0.  The one allowance: where float
arithmetic makes a NaN, any NaN is accepted (the sign and payload of a computed NaN are not specified)."""
import math
import os
import struct
import sys
from collections import OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _expr_sim as sim  # noqa: E402
import test_expr_random as TR  # noqa: E402
from test_expr_compiler import _random, _same, _table  # noqa: E402

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import expr as X  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import SelectColumns, col, functions as ff  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.table import B200Table, expr_type  # noqa: E402
from oracle import expressions as OX  # noqa: E402
from oracle import window as W  # noqa: E402

DEV = torch.device("cuda", 0)
M64 = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
N, C, I, R, NUL = K.XK_NONE, K.XK_COL, K.XK_IMM, K.XK_REG, K.XK_NULL
NP_STORAGE = {t: np.dtype(str(d).replace("torch.", "")) for t, d in K.EXPR_STORAGE.items()}
NP_VALUE = {K.T_I8: np.int8, K.T_I16: np.int16, K.T_I32: np.int32, K.T_I64: np.int64, K.T_U8: np.uint8,
            K.T_U16: np.uint16, K.T_U32: np.uint32, K.T_F16: np.float16, K.T_F32: np.float32, K.T_F64: np.float64}
FLOAT_T = (K.T_F16, K.T_F32, K.T_F64)


def fbits(v: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def bfloat(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b & M64))[0]


def sgn(v: int) -> int:
    v &= M64
    return v - (1 << 64) if v >> 63 else v


def f2i(v: float) -> int:
    """FB_X_F2I: truncate toward zero, saturate outside int64, NaN -> INT64_MIN (what the H100 does)."""
    if math.isnan(v):
        return I64_MIN
    if v >= 2.0 ** 63:
        return I64_MAX
    if v < -2.0 ** 63:
        return I64_MIN
    return math.trunc(v)


def run_device(n, cols, program, out_types, want_valid=None):
    """cols: [(numpy storage array, K8 type, validity uint8 array or None)] -> numpy outputs / validity."""
    want_valid = want_valid or [True] * len(out_types)
    dc = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a, _, _ in cols]
    dv = [None if v is None else torch.from_numpy(v).to(DEV) for _, _, v in cols]
    outs, valids = K.eval_expr(n, DEV, dc, dv, program, [K.EXPR_STORAGE[t] for t in out_types], want_valid,
                               col_types=[t for _, t, _ in cols], out_types=out_types)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs], [None if v is None else v.cpu().numpy() for v in valids]


def run_model(n, cols, program, out_types):
    return sim.run(n, [a for a, _, _ in cols], [v for _, _, v in cols], program, out_types,
                   col_types=[t for _, t, _ in cols])


def assert_same_as_model(n, cols, program, out_types, f64_bits=False):
    """``f64_bits``: the int64 outputs hold float64 bits, so two NaNs of any sign and payload are equal."""
    got, gv = run_device(n, cols, program, out_types)
    want, wv = run_model(n, cols, program, out_types)
    for o, (g, w, a, b) in enumerate(zip(got, want, gv, wv)):
        assert g.dtype == w.dtype, o
        assert np.array_equal(a, b), f"output {o}: validity differs from the model"
        tp = K.T_F64 if f64_bits else out_types[o]
        bad = np.flatnonzero((g != w) & ~(_isnan(g, tp) & _isnan(w, tp)))
        assert bad.size == 0, f"output {o}: rows {bad[:8]} differ from the model: {g[bad[:8]]} vs {w[bad[:8]]}"
    return got, gv


def _isnan(a, tp):
    if tp in FLOAT_T:
        return np.isnan(a.view(NP_VALUE[tp]))
    return np.zeros(a.shape, dtype=bool)


# ---- 1. every opcode x every operand kind, against Python ints and math -------------------------------
INT_EDGES = [I64_MIN, I64_MIN + 1, I64_MAX, -1, 0, 1, 2, -7, 1000, (1 << 53) + 1, -(1 << 53) - 1, 1 << 62]
F_EDGES = [0.0, -0.0, math.inf, -math.inf, 5e-324, -2.2250738585072e-309, 2.0 ** 53 - 1, 2.0 ** 53 + 2,
           2.0 ** 63, -2.0 ** 63, 1e300, -1e300, 1.5, -2.5, 0.1, 7.0]
NAN_BITS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000123, 0xFFFC00000000ABCD]  # +-qNaN, sNaN, payload
FLOAT_EDGE_BITS = [fbits(v) for v in F_EDGES] + NAN_BITS

UNARY = [K.X_I2F, K.X_F2I, K.X_NEG_I, K.X_NEG_F, K.X_NOT, K.X_IS_NULL, K.X_NOT_NULL, K.X_TOBOOL_I, K.X_TOBOOL_F]
INT_OPS = [K.X_ADD_I, K.X_SUB_I, K.X_RSUB_I, K.X_MUL_I, K.X_LT_I, K.X_LE_I, K.X_GT_I, K.X_GE_I, K.X_EQ_I, K.X_NE_I]
F_OPS = [K.X_ADD_F, K.X_SUB_F, K.X_RSUB_F, K.X_MUL_F, K.X_DIV_F, K.X_RDIV_F,
         K.X_LT_F, K.X_LE_F, K.X_GT_F, K.X_GE_F, K.X_EQ_F, K.X_NE_F]
LOGIC_OPS = [K.X_AND, K.X_OR, K.X_COALESCE, K.X_RCOALESCE, K.X_MOV]
F_ARITH = {K.X_ADD_F, K.X_SUB_F, K.X_RSUB_F, K.X_MUL_F, K.X_DIV_F, K.X_RDIV_F}


def _fdiv(x: float, y: float) -> float:
    if y != 0.0 or math.isnan(y):
        return x / y
    if x == 0.0 or math.isnan(x):
        return math.nan
    return math.copysign(math.inf, x) * math.copysign(1.0, y)


def ref_op(op: int, x: int, xv: bool, y: int, yv: bool):
    """(value bits, valid) of ``acc op B`` on canonical 64-bit values, in plain Python."""
    xs, ys, xf, yf = sgn(x), sgn(y), bfloat(x), bfloat(y)
    if op == K.X_MOV:
        return y, yv
    if op == K.X_I2F:
        return fbits(float(xs)), xv
    if op == K.X_F2I:
        return f2i(xf) & M64, xv
    if op == K.X_NEG_I:
        return -xs & M64, xv
    if op == K.X_NEG_F:
        return x ^ (1 << 63), xv
    if op == K.X_NOT:
        return int(x == 0), xv
    if op == K.X_IS_NULL:
        return int(not xv), True
    if op == K.X_NOT_NULL:
        return int(xv), True
    if op == K.X_TOBOOL_I:
        return int(x != 0), xv
    if op == K.X_TOBOOL_F:
        return int(xf != 0.0), xv
    if op == K.X_AND:  # Kleene: FALSE wins over NULL
        if (xv and x == 0) or (yv and y == 0):
            return 0, True
        return (1, True) if xv and yv else (0, False)
    if op == K.X_OR:  # Kleene: TRUE wins over NULL
        if (xv and x != 0) or (yv and y != 0):
            return 1, True
        return (0, True) if xv and yv else (0, False)
    if op == K.X_COALESCE:
        return (x if xv else y), xv or yv
    if op == K.X_RCOALESCE:
        return (y if yv else x), xv or yv
    fn = {
        K.X_ADD_I: lambda: (xs + ys) & M64, K.X_SUB_I: lambda: (xs - ys) & M64, K.X_RSUB_I: lambda: (ys - xs) & M64,
        K.X_MUL_I: lambda: (xs * ys) & M64,
        K.X_LT_I: lambda: int(xs < ys), K.X_LE_I: lambda: int(xs <= ys), K.X_GT_I: lambda: int(xs > ys),
        K.X_GE_I: lambda: int(xs >= ys), K.X_EQ_I: lambda: int(xs == ys), K.X_NE_I: lambda: int(xs != ys),
        K.X_ADD_F: lambda: fbits(xf + yf), K.X_SUB_F: lambda: fbits(xf - yf), K.X_RSUB_F: lambda: fbits(yf - xf),
        K.X_MUL_F: lambda: fbits(xf * yf), K.X_DIV_F: lambda: fbits(_fdiv(xf, yf)),
        K.X_RDIV_F: lambda: fbits(_fdiv(yf, xf)),
        K.X_LT_F: lambda: int(xf < yf), K.X_LE_F: lambda: int(xf <= yf), K.X_GT_F: lambda: int(xf > yf),
        K.X_GE_F: lambda: int(xf >= yf), K.X_EQ_F: lambda: int(xf == yf), K.X_NE_F: lambda: int(xf != yf),
    }[op]
    return fn(), xv and yv


def _check_rows(op, got, gv, xs, xv, ys, yv, what):
    for r, (x, a, y, b) in enumerate(zip(xs, xv, ys, yv)):
        v, ok = ref_op(op, x, bool(a), y, bool(b))
        g = int(got[r]) & M64
        assert bool(gv[r]) == ok, f"{what}: op {op} row {r} x={x:#x} y={y:#x}: validity {gv[r]} != {ok}"
        want = v if ok else 0
        if ok and op in F_ARITH and math.isnan(bfloat(v)):
            assert math.isnan(bfloat(g)), f"{what}: op {op} x={x:#x} y={y:#x}: {g:#x} is not NaN"
        else:
            assert g == want, f"{what}: op {op} x={x:#x} y={y:#x}: {g:#x} != {want:#x}"


def _pairs(edges_a, edges_b):
    xs = [a & M64 for a in edges_a for _ in edges_b]
    ys = [b & M64 for _ in edges_a for b in edges_b]
    n = len(xs)
    # validity: every (valid, valid), (NULL, valid), (valid, NULL), (NULL, NULL) combination appears for each pair
    xs, ys = xs * 4, ys * 4
    xv = np.repeat([1, 0, 1, 0], n).astype(np.uint8)
    yv = np.repeat([1, 1, 0, 0], n).astype(np.uint8)
    return np.array(xs, dtype=np.uint64).view(np.int64), xv, np.array(ys, dtype=np.uint64).view(np.int64), yv


def _edges_for(op):
    if op in F_OPS or op in (K.X_F2I, K.X_NEG_F, K.X_TOBOOL_F):
        return FLOAT_EDGE_BITS
    if op in LOGIC_OPS:
        return [0, 1, 2, fbits(-0.0)] if op in (K.X_AND, K.X_OR) else INT_EDGES + NAN_BITS[:2]
    return INT_EDGES


@pytest.mark.parametrize("op", UNARY + INT_OPS + F_OPS + LOGIC_OPS)
def test_every_opcode_with_every_operand_kind(op):
    edges = _edges_for(op)
    x, xv, y, yv = _pairs(edges, edges)
    n = len(x)
    ones = np.ones(n, dtype=np.uint8)
    cols = [(x, K.T_I64, xv), (y, K.T_I64, yv), (y, K.T_I64, None)]
    if op in UNARY:
        prog = [(K.X_MOV, C, 0, 0, 0), (op, N, 0, 0, 0), (K.X_OUT, N, 0, 0, 0)]
        got, gv = assert_same_as_model(n, cols, prog, [K.T_I64])
        _check_rows(op, got[0], gv[0], x.view(np.uint64).tolist(), xv, [0] * n, ones, "unary")
        return
    kinds = {  # operand kind -> (program, B values, B validity)
        "col+valid": ([(K.X_MOV, C, 0, 0, 0), (op, C, 1, 0, 0), (K.X_OUT, N, 0, 0, 0)], y, yv),
        "col": ([(K.X_MOV, C, 0, 0, 0), (op, C, 2, 0, 0), (K.X_OUT, N, 0, 0, 0)], y, ones),
        "reg": ([(K.X_MOV, C, 1, 0, 0), (K.X_ST, N, 3, 0, 0), (K.X_MOV, C, 0, 0, 0), (op, R, 3, 0, 0),
                 (K.X_OUT, N, 0, 0, 0)], y, yv),
        "null": ([(K.X_MOV, C, 0, 0, 0), (op, NUL, 0, 0, 0), (K.X_OUT, N, 0, 0, 0)], np.zeros(n, np.int64),
                 np.zeros(n, np.uint8)),
    }
    if op in F_OPS:  # integer operands converted on the way in, from a column and from a temporary
        ints = np.array([INT_EDGES[i % len(INT_EDGES)] for i in range(n)], dtype=np.int64)
        cols.append((ints, K.T_I64, yv))
        conv = np.array([fbits(float(v)) for v in ints.tolist()], dtype=np.uint64).view(np.int64)
        kinds["col+i2f"] = ([(K.X_MOV, C, 0, 0, 0), (op, C, 3, K.XF_B_I2F, 0), (K.X_OUT, N, 0, 0, 0)], conv, yv)
        kinds["reg+i2f"] = ([(K.X_MOV, C, 3, 0, 0), (K.X_ST, N, 0, 0, 0), (K.X_MOV, C, 0, 0, 0),
                             (op, R, 0, K.XF_B_I2F, 0), (K.X_OUT, N, 0, 0, 0)], conv, yv)
    for kind, (prog, bvals, bvalid) in kinds.items():
        got, gv = assert_same_as_model(n, cols, prog, [K.T_I64], f64_bits=op in F_ARITH)
        _check_rows(op, got[0], gv[0], x.view(np.uint64).tolist(), xv, bvals.view(np.uint64).tolist(), bvalid, kind)
    # immediates: 16 per launch, one output each
    for lo in range(0, len(edges), 16):
        imms = edges[lo:lo + 16]
        prog = []
        for o, v in enumerate(imms):
            prog += [(K.X_MOV, C, 0, 0, 0), (op, I, 0, 0, v & M64), (K.X_OUT, N, o, 0, 0)]
        got, gv = assert_same_as_model(n, cols, prog, [K.T_I64] * len(imms), f64_bits=op in F_ARITH)
        for o, v in enumerate(imms):
            _check_rows(op, got[o], gv[o], x.view(np.uint64).tolist(), xv, [v & M64] * n, ones, f"imm {v:#x}")


def test_f2i_saturates_and_maps_nan_to_int64_min():
    """FB_X_F2I on the device: the rule tests/_expr_sim.py models (DESIGN.md §7e)."""
    vals = [math.inf, -math.inf, math.nan, -math.nan, 1e300, -1e300, 2.0 ** 63, -2.0 ** 63, 2.0 ** 63 - 1024,
            -2.5, 2.5, -0.0]
    x = np.array(vals, dtype=np.float64)
    got, _ = run_device(len(x), [(x, K.T_F64, None)], [(K.X_MOV, C, 0, 0, 0), (K.X_F2I, N, 0, 0, 0),
                                                        (K.X_OUT, N, 0, 0, 0)], [K.T_I64])
    assert got[0].tolist() == [I64_MAX, I64_MIN, I64_MIN, I64_MIN, I64_MAX, I64_MIN, I64_MAX, I64_MIN, (1 << 63) - 1024,
                               -2, 2, 0]
    assert sim.f2i(x).tolist() == got[0].tolist()


# ---- 2. every input storage type x every output type ------------------------------------------------
ALL_T = [K.T_I8, K.T_I16, K.T_I32, K.T_I64, K.T_U8, K.T_U16, K.T_U32, K.T_F16, K.T_F32, K.T_F64]


def _edge_column(tp):
    """Edge values of K8 type ``tp``: (numpy array of the value type, exact Python values)."""
    vt = NP_VALUE[tp]
    if tp in FLOAT_T:
        fi = np.finfo(vt)
        v = [0.0, -0.0, 1.0, -1.5, float(fi.max), -float(fi.max), float(fi.smallest_subnormal),
             -float(fi.smallest_normal), math.inf, -math.inf, math.nan, 0.1, 65504.0 if tp != K.T_F16 else 0.25,
             3.0e9, -2049.0, 2.0 ** 63]
        if tp == K.T_F64:  # values a float16 / float32 store has to round, ties included
            v += [1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 65520.0, 65519.99, 2.0 ** -25, 3 * 2.0 ** -26,
                  1.0 + 2.0 ** -24, 1e-46, 3.4028235677973366e38]
        a = np.array(v, dtype=np.float64).astype(vt)
        return a, [float(t) for t in a.tolist()]
    ii = np.iinfo(vt)
    v = sorted({ii.min, ii.max, 0, 1, ii.max // 2 + 1, ii.max // 2, -1 if ii.min < 0 else 2, 100})
    a = np.array(v, dtype=vt)
    return a, [int(t) for t in a.tolist()]


def _expected_store(values, valid, in_float, out_tp):
    """What OUT to ``out_tp`` stores after MOV + the class conversion the compiler emits."""
    vt = NP_VALUE[out_tp]
    if out_tp in FLOAT_T:
        f = np.array([float(v) if ok else 0.0 for v, ok in zip(values, valid)], dtype=np.float64)
        return f.astype(vt).view(NP_STORAGE[out_tp])
    i = [(f2i(v) if in_float else v) if ok else 0 for v, ok in zip(values, valid)]
    return np.array(i, dtype=np.int64).astype(vt).view(NP_STORAGE[out_tp])


@pytest.mark.parametrize("in_tp", ALL_T)
def test_every_storage_type_into_every_output_type(in_tp):
    a, values = _edge_column(in_tp)
    n = len(a)
    valid = (np.arange(n) % 5 != 3).astype(np.uint8)
    in_float = in_tp in FLOAT_T
    prog = []
    for o, out_tp in enumerate(ALL_T):
        conv = []
        if in_float and out_tp not in FLOAT_T:
            conv = [(K.X_F2I, N, 0, 0, 0)]
        elif not in_float and out_tp in FLOAT_T:
            conv = [(K.X_I2F, N, 0, 0, 0)]
        prog += [(K.X_MOV, C, 0, 0, 0)] + conv + [(K.X_OUT, N, o, 0, 0)]
    cols = [(a.view(NP_STORAGE[in_tp]), in_tp, valid)]
    got, gv = assert_same_as_model(n, cols, prog, ALL_T)
    for o, out_tp in enumerate(ALL_T):
        want = _expected_store(values, valid, in_float, out_tp)
        assert got[o].dtype == want.dtype
        same = (got[o] == want) | (_isnan(got[o], out_tp) & _isnan(want, out_tp))
        assert same.all(), f"{in_tp} -> {out_tp}: {got[o][~same]} != {want[~same]} (values {np.array(values)[~same]})"
        assert np.array_equal(gv[o], valid)


def test_unsigned_and_half_columns_are_read_by_value():
    u = np.array([1, 2 ** 31 - 1, 2 ** 31, 3_000_000_000, 2 ** 32 - 1], dtype=np.uint32)
    h = np.array([1.5, -2.0, 0.25, -0.0, 65504], dtype=np.float16)
    cols = [(u.view(np.int32), K.T_U32, None), (h.view(np.int16), K.T_F16, None)]
    prog = [(K.X_MOV, C, 0, 0, 0), (K.X_ADD_I, I, 0, 0, 1), (K.X_OUT, N, 0, 0, 0),
            (K.X_MOV, C, 0, 0, 0), (K.X_GT_I, I, 0, 0, 5), (K.X_OUT, N, 1, 0, 0),
            (K.X_MOV, C, 1, 0, 0), (K.X_MUL_F, I, 0, 0, fbits(2.0)), (K.X_OUT, N, 2, 0, 0),
            (K.X_MOV, C, 1, 0, 0), (K.X_LT_F, I, 0, 0, fbits(0.0)), (K.X_OUT, N, 3, 0, 0)]
    got, _ = assert_same_as_model(5, cols, prog, [K.T_I64, K.T_U8, K.T_F64, K.T_U8])
    assert got[0].tolist() == [int(v) + 1 for v in u.tolist()]
    assert got[1].tolist() == [0, 1, 1, 1, 1]
    assert got[2].tolist() == [3.0, -4.0, 0.5, -0.0, 131008.0]
    assert got[3].tolist() == [0, 1, 0, 0, 0]


# ---- 3. sizes: tile edges and the grid-stride loop, all four temporaries live -----------------------
def _sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    g = 3 * sms * 2048
    return [0, 1, 2047, 2048, 2049, g - 1, g + 1, 5_000_011]


FOUR_TEMPS = [
    (K.X_MOV, C, 0, 0, 0), (K.X_ST, N, 0, 0, 0),                                   # t0 = a (int32)
    (K.X_MOV, C, 1, 0, 0), (K.X_ADD_I, I, 0, 0, 1), (K.X_ST, N, 1, 0, 0),         # t1 = u + 1 (uint32)
    (K.X_MOV, C, 0, 0, 0), (K.X_MUL_I, C, 1, 0, 0), (K.X_ST, N, 2, 0, 0),         # t2 = a * u
    (K.X_MOV, C, 2, 0, 0), (K.X_COALESCE, I, 0, 0, fbits(-1.0)), (K.X_ST, N, 3, 0, 0),  # t3 = coalesce(h, -1)
    (K.X_MOV, R, 0, 0, 0), (K.X_ADD_I, R, 1, 0, 0), (K.X_SUB_I, R, 2, 0, 0), (K.X_OUT, N, 0, 0, 0),
    (K.X_MOV, R, 3, 0, 0), (K.X_MUL_F, R, 0, K.XF_B_I2F, 0), (K.X_ADD_F, R, 1, K.XF_B_I2F, 0),
    (K.X_OUT, N, 1, 0, 0),
    (K.X_MOV, R, 3, 0, 0), (K.X_GT_F, I, 0, 0, 0), (K.X_OR, R, 2, 0, 0), (K.X_OUT, N, 2, 0, 0),
]


@pytest.mark.parametrize("n", _sizes())
def test_sizes_with_four_live_temporaries(n):
    rng = np.random.default_rng(n)
    a = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
    u = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    h = rng.standard_normal(n).astype(np.float16)
    hv = (rng.random(n) > 0.2).astype(np.uint8)
    uv = (rng.random(n) > 0.1).astype(np.uint8)
    cols = [(a, K.T_I32, None), (u.view(np.int32), K.T_U32, uv), (h.view(np.int16), K.T_F16, hv)]
    got, gv = assert_same_as_model(n, cols, FOUR_TEMPS, [K.T_I64, K.T_F32, K.T_U8])
    a64, u64 = a.astype(np.int64), u.astype(np.int64)
    ok = uv.astype(bool)
    with np.errstate(over="ignore"):
        e0 = np.where(ok, a64 + (u64 + 1) - a64 * u64, 0)
    t3 = np.where(hv.astype(bool), h.astype(np.float64), -1.0)
    e1 = np.where(ok, t3 * a64.astype(np.float64) + (u64 + 1).astype(np.float64), 0.0).astype(np.float32)
    assert np.array_equal(got[0], e0) and np.array_equal(gv[0], uv)
    assert np.array_equal(got[1].view(np.int32), e1.view(np.int32)) and np.array_equal(gv[1], uv)
    # OR: TRUE wins over the NULL of a * u
    e2 = (t3 > 0) | (ok & (a64 * u64 != 0))
    assert np.array_equal(got[2], e2.astype(np.uint8))
    assert np.array_equal(gv[2].astype(bool), (t3 > 0) | ok)


# ---- 4. programs at the limits ---------------------------------------------------------------------
def test_program_at_the_limits():
    """96 instructions, 16 columns of every type, 16 outputs."""
    rng = np.random.default_rng(4)
    n = 70_001
    types = ALL_T + [K.T_I32, K.T_F64, K.T_U16, K.T_F16, K.T_I8, K.T_U32]
    cols, vals = [], []
    for j, tp in enumerate(types):
        vt = NP_VALUE[tp]
        if tp in FLOAT_T:
            v = (rng.standard_normal(n) * 100).astype(vt)
        else:
            ii = np.iinfo(vt)
            v = rng.integers(max(int(ii.min), -2 ** 40), min(int(ii.max), 2 ** 40) + 1, n).astype(vt)
        m = (rng.random(n) > 0.1).astype(np.uint8) if j % 3 == 0 else None
        cols.append((v.view(NP_STORAGE[tp]), tp, m))
        vals.append(v.astype(np.float64))
    prog, outs = [], []
    for o in range(16):
        j, k, l = o, (o + 1) % 16, (o + 5) % 16
        fl = lambda c: 0 if types[c] in FLOAT_T else K.XF_B_I2F  # noqa: E731
        prog += [(K.X_MOV, C, j, fl(j), 0), (K.X_ADD_F, C, k, fl(k), 0), (K.X_MUL_F, I, 0, 0, fbits(0.5)),
                 (K.X_SUB_F, C, l, fl(l), 0), (K.X_NEG_F, N, 0, 0, 0), (K.X_OUT, N, o, 0, 0)]
        outs.append(ALL_T[o % 10] if ALL_T[o % 10] in FLOAT_T else K.T_F64)
    assert len(prog) == K.EXPR_MAX_INS
    got, gv = assert_same_as_model(n, cols, prog, outs)
    for o in range(16):
        j, k, l = o, (o + 1) % 16, (o + 5) % 16
        ok = np.ones(n, dtype=bool)
        for c in (j, k, l):
            if cols[c][2] is not None:
                ok &= cols[c][2].astype(bool)
        e = np.where(ok, -((vals[j] + vals[k]) * 0.5 - vals[l]), 0.0).astype(NP_VALUE[outs[o]])
        assert np.array_equal(got[o], e.view(NP_STORAGE[outs[o]])), o
        assert np.array_equal(gv[o].astype(bool), ok), o
    with pytest.raises(Exception):  # one instruction more is refused before anything runs
        run_device(n, cols, prog + [(K.X_OUT, N, 0, 0, 0)], outs)


# ---- 5. the seeded random trees on the device -------------------------------------------------------
def _device_and_model(t_host: B200Table, e):
    """Compile ``e`` once; run it on the device and on the model; returns (device outputs, validity, class)."""
    prog = X._Program(t_host)
    cls, _ = prog.compile(e, top=True)
    out_tp = {"i": K.T_I64, "f": K.T_F64, "b": K.T_U8, "n": K.T_I64}[cls]
    prog.output(K.EXPR_STORAGE[out_tp], True, out_tp)
    cols = [(t_host.columns[i].numpy(), expr_type(t_host.schema.types[i]),
             None if t_host.valid[i] is None else t_host.valid[i].numpy()) for i in prog.cols]
    got, gv = assert_same_as_model(t_host.num_rows, cols, prog.ins, [out_tp])
    return got[0], gv[0], cls


def _as_series(vals, valid, cls):
    dt = {"i": "Int64", "f": "Float64", "b": "boolean", "n": "Int64"}[cls]
    arr = pd.array(vals.astype(bool) if cls == "b" else vals, dtype=dt)
    arr[valid == 0] = pd.NA
    return pd.Series(arr)


def _random_trees(t_host, pdf, seed, count, **gen):
    rng = np.random.default_rng(1000 + seed)
    checked = 0
    while checked < count:
        depth = int(rng.integers(1, 5))
        e = (TR._numeric if rng.random() < 0.5 else TR._boolean)(rng, depth, **gen)
        if TR._literal_only(e):
            continue
        e = e.alias("r")
        try:
            got, gv, cls = _device_and_model(t_host, e)
        except X._OutOfResources:
            continue
        _same(_as_series(got, gv, cls), OX.select(pdf, SelectColumns(e))["r"], str(e))
        checked += 1


@pytest.mark.parametrize("seed", range(6))
def test_random_trees_on_the_device(seed):
    """The trees of test_expr_random.py (same seeds): device == model == oracle."""
    pdf = _random(n=1500, seed=seed)
    _random_trees(_table(pdf), pdf, seed, 100)


def _all_types(n, seed, nulls=True):
    """Arrow table with a column of every storage type, and the pandas frame of their values."""
    rng = np.random.default_rng(seed)
    m = (lambda q: rng.random(n) < q) if nulls else (lambda q: None)  # noqa: E731
    ints = lambda lo, hi, dt: rng.integers(lo, hi, n, dtype=np.int64).astype(dt)  # noqa: E731
    t = pa.table({
        "i8": pa.array(ints(-128, 128, np.int8), mask=m(0.1)),
        "i16": pa.array(ints(-2 ** 15, 2 ** 15, np.int16)),
        "i32": pa.array(ints(-2 ** 31, 2 ** 31, np.int32), mask=m(0.1)),
        "i64": pa.array(ints(-2 ** 40, 2 ** 40, np.int64)),
        "u8": pa.array(ints(0, 256, np.uint8), mask=m(0.1)),
        "u16": pa.array(ints(0, 2 ** 16, np.uint16)),
        "u32": pa.array(ints(0, 2 ** 32, np.uint32), mask=m(0.1)),
        "u64": pa.array(ints(0, 2 ** 40, np.uint64)),
        "f16": pa.array((rng.standard_normal(n) * 50).astype(np.float16), mask=m(0.1)),
        "f32": pa.array((rng.standard_normal(n) * 1e3).astype(np.float32)),
        "f64": pa.array(rng.standard_normal(n) * 1e6, mask=m(0.1)),
        "b": pa.array(rng.random(n) < 0.5, mask=m(0.1)),
        "d": pa.array(ints(0, 40000, np.int32), mask=m(0.1)).cast(pa.date32()),
        "ts": pa.array(ints(0, 2 ** 40, np.int64)).cast(pa.timestamp("us")),
    })
    return t


def _value_frame(t: pa.Table) -> pd.DataFrame:
    """The columns as the engine reads them: integers, dates and timestamps as Int64, floats as Float64."""
    out = {}
    for name, c in zip(t.column_names, t.columns):
        c = c.combine_chunks()
        if pa.types.is_boolean(c.type):
            out[name] = pd.array(c.to_pylist(), dtype="boolean")
        elif pa.types.is_floating(c.type):
            out[name] = pd.array(c.cast(pa.float64()).to_pylist(), dtype="Float64")
        else:
            phys = c.cast(pa.int64()) if not (pa.types.is_date32(c.type) or pa.types.is_timestamp(c.type)) \
                else c.view(pa.int32() if pa.types.is_date32(c.type) else pa.int64()).cast(pa.int64())
            out[name] = pd.array(phys.to_pylist(), dtype="Int64")
    return pd.DataFrame(out)


NUM_ALL = ["i8", "i16", "i32", "i64", "u8", "u16", "u32", "u64", "f16", "f32", "f64", "d", "ts"]


def _host_table(t: pa.Table) -> B200Table:
    dt = B200Table.from_arrow(t, DEV)
    return B200Table(dt.schema, [c.cpu() for c in dt.columns], [None if v is None else v.cpu() for v in dt.valid])


@pytest.mark.parametrize("seed", range(3))
def test_random_trees_over_every_storage_type(seed):
    t = _all_types(1200, seed)
    _random_trees(_host_table(t), _value_frame(t), 10 + seed, 100, num_cols=NUM_ALL, bool_cols=["b"],
                  denoms=[col("f64"), col("u16") + 1, col("i32") * 2 + 1])


# ---- 6. through the engine ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _frame_of(res) -> pd.DataFrame:
    return _value_frame(res.as_arrow())


def _same_frames(got: pd.DataFrame, want: pd.DataFrame):
    assert list(got.columns) == list(want.columns)
    for c in want.columns:
        _same(got[c].reset_index(drop=True), want[c].reset_index(drop=True), c)


def test_select_filter_assign_over_every_type(engine):
    t = _all_types(5000, 7)
    pdf = _value_frame(t)
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    sel = [*[(col(c) + 1).alias(f"p_{c}") for c in NUM_ALL], *[(col(c) > 100).alias(f"g_{c}") for c in NUM_ALL],
           *[(col(c) * 0.5).alias(f"h_{c}") for c in NUM_ALL],
           (col("u32") - col("i32")).alias("ui"), (col("f16") * col("u16") + col("u8")).alias("hu"),
           ff.coalesce(col("u32"), col("i8")).alias("co"), (col("b") & (col("f16") < 0)).alias("bb")]
    _same_frames(_frame_of(fa.select(df, *sel, engine=engine, as_fugue=True)), OX.select(pdf, SelectColumns(*sel)))
    cond = (col("u32") > 2 ** 31) & ((col("f16") < 0) | col("u16").is_null() | (col("i8") < 0))
    _same_frames(_frame_of(fa.filter(df, cond, engine=engine, as_fugue=True)), OX.filter_rows(pdf, cond))
    new = dict(u2=col("u32") * 2, f3=col("f16") / 3, uu=col("u16") + col("u64"))
    _same_frames(_frame_of(fa.assign(df, engine=engine, as_fugue=True, **new)),
                 OX.assign(pdf, [e.alias(k) for k, e in new.items()]))


@pytest.mark.parametrize("to", ["int8", "int16", "int32", "uint8", "uint16", "uint32", "float16", "float32"])
def test_casts_store_by_value(engine, to):
    """``cast`` to each narrow type: integers keep their low bits, floats round to nearest even once."""
    t = _all_types(3000, 8, nulls=False)
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    srcs = ["i64", "u32", "f64", "f16"]
    res = fa.select(df, *[col(c).cast(to).alias(c) for c in srcs], engine=engine, as_fugue=True).as_arrow()
    tp = pa.type_for_alias(to)
    vt = tp.to_pandas_dtype()
    for c in srcs:
        a = t.column(c).combine_chunks()
        if pa.types.is_floating(a.type):
            v = a.cast(pa.float64()).to_numpy()
            want = v.astype(vt) if pa.types.is_floating(tp) else np.trunc(v).astype(np.int64).astype(vt)
        else:
            v = a.cast(pa.int64()).to_numpy()
            want = v.astype(np.float64).astype(vt) if pa.types.is_floating(tp) else v.astype(vt)
        got = res.column(c).combine_chunks()
        assert got.type == tp
        assert np.array_equal(got.to_numpy(zero_copy_only=False).view(f"u{np.dtype(vt).itemsize}"),
                              want.view(f"u{np.dtype(vt).itemsize}")), c


@pytest.mark.parametrize("fn", ["sum", "min", "max", "avg"])
def test_aggregate_of_every_numeric_type_matches_pandas(engine, fn):
    t = _all_types(20_000, 9)
    t = t.append_column("k", pa.array(np.random.default_rng(1).integers(0, 37, t.num_rows)))
    vals = [c for c in NUM_ALL if c not in ("d", "ts")]
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    got = {}
    for part in (vals[:6], vals[6:]):  # at most 16 accumulators per call: a value and a count per column
        aggs = {c: getattr(ff, fn)(col(c)) for c in part}
        res = fa.aggregate(df, "k", engine=engine, as_fugue=True, **aggs).as_pandas()
        res = res.sort_values("k").reset_index(drop=True)
        got.update({c: res[c] for c in part})
    pdf = _value_frame(t)
    g = pdf.groupby("k", sort=True)
    for c in vals:
        if fn == "avg":
            want = g[c].mean()
        elif fn == "sum":
            want = g[c].sum(min_count=1)
        else:
            want = getattr(g[c], fn)()
        w = want.reset_index(drop=True).to_numpy(dtype=np.float64, na_value=np.nan)
        x = got[c].to_numpy(dtype=np.float64, na_value=np.nan)
        if fn in ("min", "max") or not pa.types.is_floating(t.schema.field(c).type):
            assert np.array_equal(x, w, equal_nan=True), c
        else:  # float sums: the group-by does not add in row order
            assert np.allclose(x, w, rtol=1e-9, atol=1e-6, equal_nan=True), c


@pytest.mark.parametrize("running", [True, False])
def test_window_aggregates_of_uint32_and_float16(engine, running):
    t = _all_types(4000, 10)
    t = t.append_column("rid", pa.array(np.arange(t.num_rows))).append_column(
        "k", pa.array(np.random.default_rng(2).integers(0, 30, t.num_rows)))
    cols = [getattr(ff, fn)(col(c)).over(running=running).alias(f"{fn}_{c}")
            for fn in ("sum", "min", "max", "avg") for c in ("u32", "f16")]
    out_tp = {("sum", "u32"): "long", ("sum", "f16"): "double", ("min", "u32"): "uint", ("min", "f16"): "float16",
              ("max", "u32"): "uint", ("max", "f16"): "float16", ("avg", "u32"): "double", ("avg", "f16"): "double"}
    schema = "rid:long," + ",".join(f"{fn}_{c}:{out_tp[fn, c]}" for fn in ("sum", "min", "max", "avg")
                                    for c in ("u32", "f16"))
    presort = OrderedDict(rid=True)
    res = fa.transform(B200DataFrame(B200Table.from_arrow(t, DEV)), ColumnMap(col("rid"), *cols), schema=schema,
                       partition=PartitionSpec(by=["k"], presort="rid asc"), engine=engine, as_fugue=True).as_arrow()
    order = np.argsort(np.asarray(res.column("rid")))
    exp = W.window_map(t, ["k"], presort, [col("rid")] + cols)
    for name in res.column_names:
        g = [res.column(name)[int(i)].as_py() for i in order]
        e = exp[name]
        assert [x is None for x in g] == [x is None for x in e], name
        if name.startswith(("sum_f", "avg_")):
            assert np.allclose([x for x in g if x is not None], [x for x in e if x is not None], rtol=1e-9), name
        else:
            assert g == e, name
