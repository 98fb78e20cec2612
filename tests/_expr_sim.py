"""numpy model of the fb_eval_expr accumulator machine (include/fugue_b200.h, K8): lets the host-side
expression compiler be checked against the oracle without a GPU.  Test infrastructure only."""
import numpy as np

from fugue_b200 import kernels as K

_NP_OF_T = {K.T_I8: np.int8, K.T_I16: np.int16, K.T_I32: np.int32, K.T_I64: np.int64, K.T_U8: np.uint8,
            K.T_F32: np.float32, K.T_F64: np.float64, K.T_U16: np.uint16, K.T_U32: np.uint32, K.T_F16: np.float16}


def _to_bits(a: np.ndarray, tp: int) -> np.ndarray:
    """A column in its storage dtype, read as K8 type ``tp``: canonical 64-bit value bits."""
    a = a.view(_NP_OF_T[tp])
    if a.dtype.kind == "f":
        return a.astype(np.float64).view(np.uint64)
    return a.astype(np.int64).view(np.uint64)


def f2i(x: np.ndarray) -> np.ndarray:
    """FB_X_F2I as the H100 computes it: truncate toward zero, values outside int64 saturate to INT64_MIN /
    INT64_MAX, and NaN (any sign or payload) gives INT64_MIN."""
    x = np.asarray(x, dtype=np.float64)
    t = np.trunc(np.where(np.isnan(x), -2.0 ** 64, x))
    hi, lo = t >= 2.0 ** 63, t < -2.0 ** 63
    out = np.where(hi | lo, 0.0, t).astype(np.int64)
    out[hi], out[lo] = np.iinfo(np.int64).max, np.iinfo(np.int64).min
    return out


def _f(b):
    return b.view(np.float64)


def _fb(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def _ib(x):
    return np.asarray(x).astype(np.int64).view(np.uint64)


_T_OF_NP = {np.dtype(v): k for k, v in _NP_OF_T.items() if k not in (K.T_U16, K.T_U32, K.T_F16)}


def run(n, cols, valid, program, out_types, col_types=None):
    """cols: numpy arrays (storage dtype) read as K8 types ``col_types`` (default: the signed integer or
    float of each array's dtype); valid: uint8 arrays or None.  Returns ([values], [valid]); outputs are
    in their storage dtype (``kernels.EXPR_STORAGE``)."""
    if col_types is None:
        col_types = [_T_OF_NP[np.asarray(c).dtype] for c in cols]
    acc = np.zeros(n, dtype=np.uint64)
    accv = np.ones(n, dtype=bool)
    tmp = {}
    outs = [None] * len(out_types)
    outv = [None] * len(out_types)
    with np.errstate(all="ignore"):
        for op, kind, b, flags, imm in program:
            bv = np.ones(n, dtype=bool)
            bb = np.full(n, imm & ((1 << 64) - 1), dtype=np.uint64)
            if kind == K.XK_COL:
                bb = _to_bits(cols[b], col_types[b])
                if valid[b] is not None:
                    bv = valid[b] != 0
            elif kind == K.XK_REG:
                bb, bv = tmp[b]
            elif kind == K.XK_NULL:
                bv = np.zeros(n, dtype=bool)
            if flags & K.XF_B_I2F:
                bb = _fb(bb.view(np.int64).astype(np.float64))
            x, y = acc, bb
            xi, yi = x.view(np.int64), y.view(np.int64)
            if op == K.X_MOV:
                acc, accv = bb.copy(), bv.copy()
            elif op == K.X_ST:
                tmp[b] = (acc.copy(), accv.copy())
            elif op == K.X_OUT:
                t = out_types[b]
                vals = np.where(accv, acc, np.uint64(0))
                if t in (K.T_F16, K.T_F32, K.T_F64):
                    o = _f(vals).astype(_NP_OF_T[t])  # numpy rounds a double to nearest even once
                else:
                    o = vals.view(np.int64).astype(_NP_OF_T[t])
                outs[b] = o.view({K.T_U16: np.int16, K.T_U32: np.int32, K.T_F16: np.int16}.get(t, o.dtype))
                outv[b] = accv.astype(np.uint8)
            elif op == K.X_I2F:
                acc = _fb(xi.astype(np.float64))
            elif op == K.X_F2I:
                acc = _ib(f2i(_f(x)))
            elif op == K.X_NEG_I:
                acc = _ib(-xi)
            elif op == K.X_NEG_F:
                acc = x ^ np.uint64(1 << 63)
            elif op == K.X_NOT:
                acc = _ib(x == 0)
            elif op == K.X_IS_NULL:
                acc, accv = _ib(~accv), np.ones(n, dtype=bool)
            elif op == K.X_NOT_NULL:
                acc, accv = _ib(accv), np.ones(n, dtype=bool)
            elif op == K.X_TOBOOL_I:
                acc = _ib(x != 0)
            elif op == K.X_TOBOOL_F:
                acc = _ib(_f(x) != 0.0)
            elif op in (K.X_AND, K.X_OR):
                if op == K.X_AND:
                    fa, fb = accv & (x == 0), bv & (y == 0)
                    isf = fa | fb
                    nv = isf | (accv & bv)
                    acc = _ib(~isf & accv & bv)
                else:
                    ta, tb = accv & (x != 0), bv & (y != 0)
                    ist = ta | tb
                    nv = ist | (accv & bv)
                    acc = _ib(ist)
                accv = nv
            elif op == K.X_COALESCE:
                acc = np.where(accv, x, y)
                accv = accv | bv
            elif op == K.X_RCOALESCE:
                acc = np.where(bv, y, x)
                accv = accv | bv
            else:
                xf, yf = _f(x), _f(y)
                table = {
                    K.X_ADD_I: lambda: _ib(xi + yi), K.X_SUB_I: lambda: _ib(xi - yi), K.X_RSUB_I: lambda: _ib(yi - xi),
                    K.X_MUL_I: lambda: _ib(xi * yi),
                    K.X_ADD_F: lambda: _fb(xf + yf), K.X_SUB_F: lambda: _fb(xf - yf), K.X_RSUB_F: lambda: _fb(yf - xf),
                    K.X_MUL_F: lambda: _fb(xf * yf), K.X_DIV_F: lambda: _fb(xf / yf), K.X_RDIV_F: lambda: _fb(yf / xf),
                    K.X_LT_I: lambda: _ib(xi < yi), K.X_LE_I: lambda: _ib(xi <= yi), K.X_GT_I: lambda: _ib(xi > yi),
                    K.X_GE_I: lambda: _ib(xi >= yi), K.X_EQ_I: lambda: _ib(xi == yi), K.X_NE_I: lambda: _ib(xi != yi),
                    K.X_LT_F: lambda: _ib(xf < yf), K.X_LE_F: lambda: _ib(xf <= yf), K.X_GT_F: lambda: _ib(xf > yf),
                    K.X_GE_F: lambda: _ib(xf >= yf), K.X_EQ_F: lambda: _ib(xf == yf), K.X_NE_F: lambda: _ib(xf != yf),
                }
                acc = table[op]()
                accv = accv & bv
    return outs, outv
