"""Randomly generated expression trees: compiled programs (fugue_b200/expr.py) simulated on the CPU model of the
accumulator machine (tests/_expr_sim.py) against oracle/expressions.py.  Seeded, so every run checks the same
600 trees; complements the hand-picked list in test_expr_compiler.py.  CPU only (the -m gpu tests execute
programs from the same compiler on the device)."""
import numpy as np
import pytest

from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200.column import SelectColumns, col, functions as ff, lit, null
from oracle import expressions as OX
from test_expr_compiler import _random, _run, _same, _table

NUM_COLS = ["a", "b", "x", "y", "g"]      # int64, int32, float64 with NaN->NULL, float64, nullable int64
BOOL_COLS = ["p"]                          # nullable boolean
DENOMS = [col("y"), col("b") + 1, col("a") * 2 + 1]  # never 0


def _numeric(rng, depth, div=True, num_cols=NUM_COLS, bool_cols=BOOL_COLS, denoms=DENOMS):
    """``div=False``: no division below this node - a quotient can be +-inf, and inf -> integer has no defined
    result (pandas, the reference's evaluator, refuses it).  ``num_cols`` / ``bool_cols``: the leaves;
    ``denoms``: the denominators, expressions that are never 0."""
    cs = dict(num_cols=num_cols, bool_cols=bool_cols, denoms=denoms)
    if depth == 0 or rng.random() < 0.25:
        r = rng.random()
        if r < 0.7:
            return col(num_cols[rng.integers(len(num_cols))])
        if r < 0.85:
            return lit(int(rng.integers(-5, 6)))
        return lit(float(np.round(rng.normal() * 3, 2)))
    r = rng.random()
    if r < 0.6:
        op = rng.integers(4 if div else 3)
        l, rr = _numeric(rng, depth - 1, div, **cs), _numeric(rng, depth - 1, div, **cs)
        if op == 3:
            # denominators that are never 0: x / 0 = inf and 0 / 0 = inf - inf = NaN are where the two sides
            # legitimately part - pandas (the reference's evaluator) reads an arithmetic NaN as NULL, the device
            # keeps it a valid IEEE NaN (DESIGN.md, K8); division by zero itself is covered in test_expr_compiler
            opts = denoms[:2] + [lit(float(np.round(rng.uniform(0.5, 4), 2)))] + denoms[2:]
            rr = opts[rng.integers(len(opts))]
        return [lambda: l + rr, lambda: l - rr, lambda: l * rr, lambda: l / rr][op]()
    if r < 0.7:
        return -_numeric(rng, depth - 1, div, **cs)
    if r < 0.85:
        return ff.coalesce(_numeric(rng, depth - 1, div, **cs), _numeric(rng, depth - 1, div, **cs))
    if r < 0.93:
        to = [int, float, "long", "double"][rng.integers(4)]
        return _numeric(rng, depth - 1, div and to in (float, "double"), **cs).cast(to)
    return _boolean(rng, depth - 1, **cs).cast(int)


def _boolean(rng, depth, num_cols=NUM_COLS, bool_cols=BOOL_COLS, denoms=DENOMS):
    cs = dict(num_cols=num_cols, bool_cols=bool_cols, denoms=denoms)
    if depth == 0 or rng.random() < 0.15:
        return col(bool_cols[rng.integers(len(bool_cols))]) if rng.random() < 0.8 else lit(bool(rng.integers(2)))
    r = rng.random()
    if r < 0.45:
        l, rr = _numeric(rng, depth - 1, **cs), _numeric(rng, depth - 1, **cs)
        return [lambda: l < rr, lambda: l <= rr, lambda: l > rr, lambda: l >= rr, lambda: l == rr,
                lambda: l != rr][rng.integers(6)]()
    if r < 0.75:
        l, rr = _boolean(rng, depth - 1, **cs), _boolean(rng, depth - 1, **cs)
        return (l & rr) if rng.random() < 0.5 else (l | rr)
    if r < 0.85:
        return ~_boolean(rng, depth - 1, **cs)
    if r < 0.95:
        e = _numeric(rng, depth - 1, **cs)
        return e.is_null() if rng.random() < 0.5 else e.not_null()
    return null() & _boolean(rng, depth - 1, **cs) if rng.random() < 0.5 else _boolean(rng, depth - 1, **cs) | null()


def _literal_only(e) -> bool:
    from fugue_b200.column import column_mentions

    return len(list(column_mentions(e))) == 0


@pytest.mark.parametrize("seed", range(6))
def test_random_trees_match_oracle(seed):
    rng = np.random.default_rng(1000 + seed)
    pdf = _random(n=1500, seed=seed)
    t = _table(pdf)
    checked = skipped = 0
    while checked < 100:
        depth = int(rng.integers(1, 5))
        e = (_numeric if rng.random() < 0.5 else _boolean)(rng, depth)
        if _literal_only(e):
            continue
        e = e.alias("r")
        try:
            got, prog = _run(t, [e])
        except X._OutOfResources:       # deeper than the register file: the engine splits such trees
            skipped += 1
            continue
        assert len(prog.ins) <= K.EXPR_MAX_INS
        want = OX.select(pdf, SelectColumns(e))
        _same(got[0], want["r"], str(e))
        checked += 1
    assert skipped < 100
