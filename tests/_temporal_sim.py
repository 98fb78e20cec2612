"""numpy model of the temporal ops of fb_eval_expr (``FB_X_MULSAT_I`` ... ``FB_X_TS_ADDMON``, include/fugue_b200.h, K8)
on top of the machine model of tests/_func_sim.py.  Test infrastructure only.

The functions mirror fugue_b200/csrc/fb_expr.cu step by step on int64 arrays: sums and products wrap as the device's do,
every division floors, so the model gives the device's bits for every int64 input, also outside the calendar's exact
domain.  ``run`` takes the arguments of ``_expr_sim.run``; the program is cut at every temporal op, each piece runs in
``_func_sim.run`` with the accumulator and the temporaries passed in and out as extra int64 columns and outputs."""
import numpy as np

import _expr_sim as sim
import _func_sim as fsim
from fugue_b200 import kernels as K

I64 = np.int64
_PER_SECOND = {K.TU_DAY: 1, K.TU_S: 1, K.TU_MS: 10 ** 3, K.TU_US: 10 ** 6, K.TU_NS: 10 ** 9}
F = {n: i for i, n in enumerate(K.TIME_FIELDS)}
P = {n: i for i, n in enumerate(K.TIME_PARTS)}


def _fdiv(x, c):
    return np.floor_divide(x, I64(c))


def split_days(x, unit):
    if unit == K.TU_DAY:
        return x.copy(), np.zeros_like(x)
    s = x if unit == K.TU_S else _fdiv(x, _PER_SECOND[unit])
    days = _fdiv(s, 86400)
    return days, s - days * I64(86400)


def join_days(days, sod, unit):
    if unit == K.TU_DAY:
        return days
    return (days * I64(86400) + sod) * I64(_PER_SECOND[unit])


def is_leap(y):
    return ((y & I64(3)) == 0) & ((np.fmod(y, I64(100)) != 0) | (np.fmod(y, I64(400)) == 0))


def civil_from_days(days):
    z = days + I64(719468)
    era = _fdiv(z, 146097)
    doe = z - era * I64(146097)
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy_m = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy_m + 2) // 153
    d = doy_m - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    y = yoe + era * I64(400) + (m <= 2)
    doy = np.where(mp < 10, doy_m + 60 + is_leap(y), doy_m - 305)
    return y, m, d, doy


def days_from_civil(y, m, d):
    y = y - (m <= 2)
    era = _fdiv(y, 400)
    yoe = y - era * I64(400)
    doy_m = (153 * np.where(m > 2, m - 3, m + 9) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy_m
    return era * I64(146097) + doe - I64(719468)


def iso_weekday(days):
    t = days + I64(3)
    return t - _fdiv(t, 7) * I64(7) + 1


def ts_part(x, field, unit):
    days, sod = split_days(x, unit)
    if field == F["hour"]:
        return sod // 3600
    if field == F["minute"]:
        return sod // 60 % 60
    if field == F["second"]:
        return sod % 60
    if field == F["dow"]:
        return iso_weekday(days) % 7
    if field == F["isodow"]:
        return iso_weekday(days)
    if field in (F["week"], F["isoyear"]):
        days = days + (4 - iso_weekday(days))
    y, m, d, doy = civil_from_days(days)
    return {F["month"]: m, F["day"]: d, F["quarter"]: (m - 1) // 3 + 1, F["doy"]: doy,
            F["week"]: (doy - 1) // 7 + 1}.get(field, y)


def ts_trunc(x, part, unit):
    days, sod = split_days(x, unit)
    if part == P["minute"]:
        sod = sod - sod % 60
    elif part == P["hour"]:
        sod = sod - sod % 3600
    elif part == P["day"]:
        sod = np.zeros_like(sod)
    elif part == P["week"]:
        sod, days = np.zeros_like(sod), days - (iso_weekday(days) - 1)
    elif part != P["second"]:
        y, m, _, _ = civil_from_days(days)
        m = np.ones_like(m) if part == P["year"] else ((m - 1) // 3 * 3 + 1 if part == P["quarter"] else m)
        sod, days = np.zeros_like(sod), days_from_civil(y, m, np.ones_like(m))
    return join_days(days, sod, unit)


def ts_index(x, part, unit):
    days, sod = split_days(x, unit)
    if part == P["second"]:
        return days * I64(86400) + sod
    if part == P["minute"]:
        return days * I64(1440) + sod // 60
    if part == P["hour"]:
        return days * I64(24) + sod // 3600
    if part == P["day"]:
        return days
    if part == P["week"]:
        return _fdiv(days + I64(3), 7)
    y, m, _, _ = civil_from_days(days)
    y = y - I64(1970)
    return y if part == P["year"] else (y * I64(4) + (m - 1) // 3 if part == P["quarter"] else y * I64(12) + (m - 1))


def ts_addmon(x, n, unit):
    days, sod = split_days(x, unit)
    sub = x - join_days(days, sod, unit)
    y, m, d, _ = civil_from_days(days)
    mi = y * I64(12) + (m - 1) + n
    y2 = _fdiv(mi, 12)
    m2 = mi - y2 * I64(12) + 1
    last = np.where(m2 == 2, 28 + is_leap(y2), 30 + ((m2 + (m2 >> 3)) & 1))
    return join_days(days_from_civil(y2, m2, np.minimum(d, last)), sod, unit) + sub


def mulsat(x, b):
    out = []
    for v in x.tolist():
        out.append(min(max(v * b, -(1 << 63)), (1 << 63) - 1))
    return np.array(out, dtype=I64)


def apply(op, acc, accv, bb, bv, flags, imm):
    """One temporal op on the machine state: returns the new (acc, accv)."""
    x, y = acc.view(I64), bb.view(I64)
    with np.errstate(all="ignore"):
        if op == K.X_MULSAT_I:
            return mulsat(x, int(y[0]) if len(y) else 1).view(np.uint64), accv & bv
        if op == K.X_FLOORDIV_I:
            return np.floor_divide(x, y).view(np.uint64), accv & bv
        if op == K.X_TS_ADDMON:
            return ts_addmon(x, y, flags >> K.XF_UNIT_SHIFT).astype(I64).view(np.uint64), accv & bv
        fn = {K.X_TS_PART: ts_part, K.X_TS_TRUNC: ts_trunc, K.X_TS_INDEX: ts_index}[op]
        return fn(x, imm & 0xFF, imm >> 8).astype(I64).view(np.uint64), accv


def run(n, cols, valid, program, out_types, col_types=None):
    if col_types is None:
        col_types = [sim._T_OF_NP[np.asarray(c).dtype] for c in cols]
    nout = len(out_types)
    outs, outv = [None] * nout, [None] * nout
    acc, accv = np.zeros(n, dtype=np.uint64), np.ones(n, dtype=bool)
    regs = {}
    piece = []
    for ins in list(program) + [None]:
        if ins is not None and ins[0] < K.X_MULSAT_I:
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
        o, ov = fsim.run(n, list(cols) + [a.view(I64) for a in extra],
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
        bb, bv = fsim._operand(n, cols, valid, col_types, regs, kind, b, flags, imm)
        acc, accv = apply(op, acc, accv, bb, bv, flags, imm & ((1 << 64) - 1))
        piece = []
    return outs, outv
