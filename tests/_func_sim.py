"""numpy model of the scalar-function ops of fb_eval_expr (``FB_X_SEL`` ... ``FB_X_LEAST_F``, include/fugue_b200.h, K8)
on top of the machine model of tests/_expr_sim.py and the lookup of tests/_lookup_sim.py.  Test infrastructure only.

``run`` takes the arguments of ``_expr_sim.run``.  As in ``_lookup_sim``, the program is cut at every op the base model
does not know; each piece runs in ``_expr_sim.run`` with the accumulator and the temporaries passed in and out as extra
int64 columns and outputs, and the op itself is applied here between two pieces.  The float functions use numpy's
float64 ``fmod``, ``floor``, ``ceil``, ``sqrt`` (all exact or correctly rounded, as on the device); ``exp``, ``log``,
``log10`` and ``power`` are numpy's, which may differ from CUDA's in the last bits: tests compare those within the
ulp bounds of the CUDA Programming Guide."""
import numpy as np

import _expr_sim as sim
import _lookup_sim as lsim
from fugue_b200 import kernels as K

_INT64_MIN = np.int64(-(1 << 63))
_POW10_I = [10 ** d for d in range(19)]


def _operand(n, cols, valid, col_types, regs, kind, b, flags, imm):
    bv = np.ones(n, dtype=bool)
    bb = np.full(n, imm & ((1 << 64) - 1), dtype=np.uint64)
    if kind == K.XK_COL:
        bb = sim._to_bits(cols[b], col_types[b])
        if valid[b] is not None:
            bv = valid[b] != 0
    elif kind == K.XK_REG:
        bb, bv = regs[b]
    elif kind == K.XK_NULL:
        bv = np.zeros(n, dtype=bool)
    if kind in (K.XK_NONE, K.XK_NULL):
        bb = np.zeros(n, dtype=np.uint64)
    if flags & K.XF_B_I2F:
        bb = sim._fb(bb.view(np.int64).astype(np.float64))
    return bb, bv


def mod_i(x: np.ndarray, y: np.ndarray):
    """Truncated remainder of int64 bits; (values, ok) with ok False where y = 0."""
    xi, yi = x.view(np.int64), y.view(np.int64)
    safe = np.where((yi == 0) | (yi == -1), np.int64(1), yi)
    r = np.fmod(xi, safe)  # C's %: the sign of x
    r = np.where((yi == 0) | (yi == -1), np.int64(0), r)
    return r.view(np.uint64), yi != 0


def mod_f(x: np.ndarray, y: np.ndarray):
    xf, yf = sim._f(x), sim._f(y)
    r = np.fmod(xf, yf)
    ok = (yf != 0.0) & ~(np.isnan(r) & ~np.isnan(xf) & ~np.isnan(yf))
    return sim._fb(r), ok


def round_f(x: np.ndarray, d: int) -> np.ndarray:
    """DuckDB's ROUND of float64 bits: C round (half away from zero) of x * 10^d, divided back; x when not finite."""
    xf = sim._f(x)

    def cround(s):
        t = np.trunc(s)
        return np.where(np.abs(s - t) >= 0.5, t + np.copysign(1.0, s), t)  # s - t is exact for |s| < 2^52

    if d == 0:
        return sim._fb(cround(xf))
    p = float(10 ** abs(d))
    s = xf * p if d > 0 else xf / p
    r = cround(s) / p if d > 0 else cround(s) * p
    return sim._fb(np.where(np.isfinite(s), r, xf))


def round_i(x: np.ndarray, d: int) -> np.ndarray:
    p = _POW10_I[-d]
    out = []
    for v in x.view(np.int64).tolist():
        r = abs(v) % p
        q = abs(v) - r + (p if 2 * r >= p else 0)
        q = q if v >= 0 else -q
        out.append(q & ((1 << 64) - 1))
    return np.array(out, dtype=np.uint64)


def total_key(x: np.ndarray) -> np.ndarray:
    s = x.view(np.int64)
    return np.where(s >= 0, s, s ^ np.int64(0x7FFFFFFFFFFFFFFF))


def _float_fn(fn, x: np.ndarray, accv: np.ndarray):
    xf = sim._f(x)
    r = fn(xf)
    return sim._fb(r), accv & ~(np.isnan(r) & ~np.isnan(xf))


_UNARY_F = {K.X_SQRT: np.sqrt, K.X_EXP: np.exp, K.X_LN: np.log, K.X_LOG10: np.log10}


def apply(op, acc, accv, bb, bv, flags, imm, regs):
    """One scalar-function op on the machine state: returns the new (acc, accv)."""
    if op == K.X_SEL:
        c, cv = regs[flags >> K.XF_COND_SHIFT]
        t = cv & (c != 0)
        return np.where(t, acc, bb), np.where(t, accv, bv)
    if op in (K.X_MOD_I, K.X_RMOD_I):
        r, ok = mod_i(acc, bb) if op == K.X_MOD_I else mod_i(bb, acc)
        return r, accv & bv & ok
    if op in (K.X_MOD_F, K.X_RMOD_F):
        r, ok = mod_f(acc, bb) if op == K.X_MOD_F else mod_f(bb, acc)
        return r, accv & bv & ok
    if op == K.X_ABS_I:
        xi = acc.view(np.int64)
        return np.where(xi < 0, (np.uint64(0) - acc), acc), accv
    if op == K.X_ABS_F:
        return acc & np.uint64(0x7FFFFFFFFFFFFFFF), accv
    if op == K.X_FLOOR_F:
        return sim._fb(np.floor(sim._f(acc))), accv
    if op == K.X_CEIL_F:
        return sim._fb(np.ceil(sim._f(acc))), accv
    d = imm - (1 << 64) if imm >= (1 << 63) else imm
    if op == K.X_ROUND_F:
        return round_f(acc, d), accv
    if op == K.X_ROUND_I:
        return round_i(acc, d), accv
    if op in _UNARY_F:
        return _float_fn(_UNARY_F[op], acc, accv)
    if op in (K.X_POW, K.X_RPOW):
        xf, yf = (sim._f(acc), sim._f(bb)) if op == K.X_POW else (sim._f(bb), sim._f(acc))
        r = np.power(xf, yf)
        return sim._fb(r), accv & bv & ~(np.isnan(r) & ~np.isnan(xf) & ~np.isnan(yf))
    if op in (K.X_GREATEST_I, K.X_LEAST_I, K.X_GREATEST_F, K.X_LEAST_F):
        if op in (K.X_GREATEST_I, K.X_LEAST_I):
            ka, kb = acc.view(np.int64), bb.view(np.int64)
        else:
            ka, kb = total_key(acc), total_key(bb)
        better = kb > ka if op in (K.X_GREATEST_I, K.X_GREATEST_F) else kb < ka
        take = bv & (~accv | better)
        return np.where(take, bb, acc), accv | bv
    raise AssertionError(f"op {op} is not a scalar-function op")


def run(n, cols, valid, program, out_types, col_types=None):
    if col_types is None:
        col_types = [sim._T_OF_NP[np.asarray(c).dtype] for c in cols]
    nout = len(out_types)
    outs, outv = [None] * nout, [None] * nout
    acc, accv = np.zeros(n, dtype=np.uint64), np.ones(n, dtype=bool)
    regs = {}
    piece = []
    for ins in list(program) + [None]:
        if ins is not None and ins[0] < K.X_SEL:
            piece.append(ins)
            continue
        extra = [acc] + [regs[r][0] for r in sorted(regs)]
        extra_v = [accv] + [regs[r][1] for r in sorted(regs)]
        base = len(cols)
        pre = []
        for j, r in enumerate(sorted(regs)):
            pre += [(K.X_MOV, K.XK_COL, base + 1 + j, 0, 0), (K.X_ST, K.XK_NONE, r, 0, 0)]
        pre.append((K.X_MOV, K.XK_COL, base, 0, 0))
        stored = sorted(set(regs) | {b for op, _, b, _, _ in piece if op == K.X_ST})
        post = [(K.X_OUT, K.XK_NONE, nout, 0, 0)]
        for j, r in enumerate(stored):
            post += [(K.X_MOV, K.XK_REG, r, 0, 0), (K.X_OUT, K.XK_NONE, nout + 1 + j, 0, 0)]
        o, ov = lsim.run(n, list(cols) + [a.view(np.int64) for a in extra],
                         list(valid) + [v.astype(np.uint8) for v in extra_v], pre + piece + post,
                         list(out_types) + [K.T_I64] * (1 + len(stored)), list(col_types) + [K.T_I64] * len(extra))
        for b in range(nout):
            if o[b] is not None:
                outs[b], outv[b] = o[b], ov[b]
        acc, accv = o[nout].view(np.uint64), ov[nout] != 0
        regs = {r: (o[nout + 1 + j].view(np.uint64), ov[nout + 1 + j] != 0) for j, r in enumerate(stored)}
        if ins is None:
            break
        op, kind, b, flags, imm = ins
        bb, bv = _operand(n, cols, valid, col_types, regs, kind, b, flags, imm)
        with np.errstate(all="ignore"):
            acc, accv = apply(op, acc, accv, bb, bv, flags, imm & ((1 << 64) - 1), regs)
        acc = acc.astype(np.uint64)
        piece = []
    return outs, outv
