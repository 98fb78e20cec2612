"""numpy model of FB_X_LOOKUP (include/fugue_b200.h, K8) on top of the machine model of tests/_expr_sim.py.
Test infrastructure only.

``run`` takes the arguments of ``_expr_sim.run``.  The program is cut at every ``X_LOOKUP``; each piece runs in
``_expr_sim.run`` with the machine state it needs passed in and out through extra int64 columns and outputs (the
accumulator and every temporary written so far, each with its validity), and the lookup itself is applied here
between two pieces.  Values under NULL are never observable in K8, so passing them as 0 changes nothing."""
import numpy as np

import _expr_sim as sim
from fugue_b200 import kernels as K


def lookup(acc: np.ndarray, accv: np.ndarray, table: np.ndarray, valid, nent: int):
    """``acc <- table[acc]``: NULL for a NULL accumulator or an entry number outside [0, nent)."""
    ok = accv & (acc < np.uint64(max(nent, 0)))
    e = np.where(ok, acc, np.uint64(0)).astype(np.int64)
    tab = np.append(table, np.uint64(0))  # a spare entry: an empty table still has an index 0
    hit = np.ones(len(acc), dtype=bool) if valid is None else np.append(valid != 0, False)[e]
    return np.where(ok, tab[e], np.uint64(0)), ok & hit


def run(n, cols, valid, program, out_types, col_types=None):
    if col_types is None:
        col_types = [sim._T_OF_NP[np.asarray(c).dtype] for c in cols]
    nout = len(out_types)
    outs, outv = [None] * nout, [None] * nout
    acc, accv = np.zeros(n, dtype=np.uint64), np.ones(n, dtype=bool)
    regs = {}  # temporary -> (values, validity)
    piece = []
    for ins in list(program) + [None]:
        if ins is not None and ins[0] != K.X_LOOKUP:
            piece.append(ins)
            continue
        # state in: the accumulator and the temporaries as extra columns; state out: as extra outputs
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
        o, ov = sim.run(n, list(cols) + [a.view(np.int64) for a in extra],
                        list(valid) + [v.astype(np.uint8) for v in extra_v], pre + piece + post,
                        list(out_types) + [K.T_I64] * (1 + len(stored)), list(col_types) + [K.T_I64] * len(extra))
        for b in range(nout):
            if o[b] is not None:
                outs[b], outv[b] = o[b], ov[b]
        acc, accv = o[nout].view(np.uint64), ov[nout] != 0
        regs = {r: (o[nout + 1 + j].view(np.uint64), ov[nout + 1 + j] != 0) for j, r in enumerate(stored)}
        if ins is None:
            break
        _, _, b, _, imm = ins
        acc, accv = lookup(acc, accv, sim._to_bits(cols[b], col_types[b]), valid[b], imm)
        piece = []
    return outs, outv
