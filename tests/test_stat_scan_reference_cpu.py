"""The integer reference of the statistics scans (tests/_stat_scan_reference.py) against the Fraction oracles
(oracle.moments, oracle.comoments, oracle.shape_moments) on small random inputs with NULLs, empty segments and
non-finite values: counts exactly, central sums exactly, and every word rounded once."""
import math
from fractions import Fraction
from typing import List, Optional

import numpy as np
import pytest

import _stat_scan_reference as R
from oracle import comoments as OC
from oracle import moments as OM
from oracle import shape_moments as OS

SPECIAL = [math.inf, -math.inf, math.nan]


def _offsets(rng: np.random.Generator, n: int) -> np.ndarray:
    cuts = np.sort(rng.integers(0, n + 1, max(n // 8, 1)))
    return np.sort(np.concatenate([[0, 0], cuts, cuts[:3], [n, n]])).astype(np.int64)  # empty segments too


def _column(rng: np.random.Generator, n: int, shift: float, kmax: int, special: float):
    k = rng.integers(-kmax + 1, kmax, n)
    if n:
        k[rng.random(n) < 0.1] = kmax - 1  # the largest |k|, both signs
        k[rng.random(n) < 0.1] = -kmax + 1
    x = R.dyadic(k, shift)
    sp = rng.random(n) < special
    x[sp] = rng.choice(SPECIAL, int(sp.sum()))
    valid = (rng.random(n) > 0.15).astype(np.uint8)
    return x, valid


def _values(x: np.ndarray, valid: Optional[np.ndarray]) -> List[Optional[float]]:
    return [float(v) if valid is None or ok else None for v, ok in zip(x.tolist(), (valid if valid is not None
                                                                                   else np.ones(len(x))).tolist())]


def _same(got: float, want: Optional[float]) -> bool:
    want = 0.0 if want is None else float(want)
    return (math.isnan(got) and math.isnan(want)) or got == want


SEEDS = range(6)


@pytest.mark.parametrize("seed", SEEDS)
def test_moments_match_the_fraction_oracle(seed):
    rng = np.random.default_rng(seed)
    n = 400
    x, valid = _column(rng, n, R.MOMENT_SHIFT, R.MOMENT_K, 0.01 if seed % 2 else 0.0)
    valid = None if seed == 0 else valid
    off = _offsets(rng, n)
    ref = R.RunningMoments(off, x, valid)
    (m2,), (b,) = ref.want(np.arange(n))
    for a, e in zip(off[:-1], off[1:]):
        vals = _values(x[a:e], None if valid is None else valid[a:e])
        for i, (m, want) in enumerate(OM.running_moments(vals)):
            r = a + i
            assert ref.count[r] == m
            assert _same(m2[r], want), (r, m2[r], want)
            finite = [v for v in vals[:i + 1] if v is not None]
            if m and not math.isnan(m2[r]):
                assert ref.m2_fraction(r) == OM.exact_m2(finite)
                sx2 = float(sum(Fraction(v) ** 2 for v in finite))
                assert b[r] == pytest.approx(4 * m * R.U * math.sqrt(sx2 * m2[r]), rel=1e-12)


@pytest.mark.parametrize("seed", SEEDS)
def test_comoments_match_the_fraction_oracle(seed):
    rng = np.random.default_rng(100 + seed)
    n = 300
    x, xv = _column(rng, n, R.MOMENT_SHIFT, R.MOMENT_K, 0.01 if seed % 2 else 0.0)
    y, yv = _column(rng, n, -2.0 ** 19, R.MOMENT_K, 0.01 if seed % 3 == 1 else 0.0)
    if seed == 0:
        yv = None
    off = _offsets(rng, n)
    ref = R.RunningCoMoments(off, x, xv, y, yv, R.MOMENT_SHIFT, -2.0 ** 19)
    words, bounds = ref.want(np.arange(n))
    for a, e in zip(off[:-1], off[1:]):
        xs, ys = _values(x[a:e], xv[a:e]), _values(y[a:e], None if yv is None else yv[a:e])
        for i, st in enumerate(OC.running_states(xs, ys)):
            r = a + i
            assert ref.count[r] == st[0]
            for w, q in zip(words, st[1:]):
                assert _same(w[r], q), (r, w[r], q)
            if st[0] and not isinstance(st[3], float):
                assert ref.state(r) == st
                pairs = OC.pair_rows(xs[:i + 1], ys[:i + 1])
                ax, ay = max(abs(p) for p, _ in pairs), max(abs(q) for _, q in pairs)
                assert bounds[0][r] == 4 * st[0] * R.U * ax and bounds[1][r] == 4 * st[0] * R.U * ay


@pytest.mark.parametrize("seed", SEEDS)
def test_shape_moments_match_the_fraction_oracle(seed):
    rng = np.random.default_rng(200 + seed)
    n = 250
    x, valid = _column(rng, n, R.SHAPE_SHIFT, R.SHAPE_K, 0.01 if seed % 2 else 0.0)
    off = _offsets(rng, n)
    ref = R.RunningShapeMoments(off, x, valid)
    words, bounds = ref.want(np.arange(n))
    for a, e in zip(off[:-1], off[1:]):
        vals = _values(x[a:e], valid[a:e])
        for i in range(e - a):
            r = a + i
            mom = OS.central_sums(vals[:i + 1])
            assert ref.count[r] == mom[0]
            nan = mom[0] > 0 and mom[1] is None
            for w, q in zip(words, mom[1:]):
                assert _same(w[r], math.nan if nan else q), (r, w[r], q)
            assert ref.central_sums(r) == mom
            if mom[1] is not None:
                # sound: never tighter than the bound evaluated over the values themselves
                finite = [v for v in vals[:i + 1] if v is not None]
                for got, want in zip(ref.bounds(r), OS.sums_bound(finite, "scan")):
                    assert got >= want * (1 - 1e-9), (r, got, want)


def test_int64_limits_are_asserted():
    off = np.array([0, 2], dtype=np.int64)
    with pytest.raises(AssertionError, match="too large"):
        R.RunningMoments(off, R.dyadic(np.array([0, R.MOMENT_K]), R.MOMENT_SHIFT), None)
    with pytest.raises(AssertionError, match="not k / 2"):
        R.RunningShapeMoments(off, np.array([64.0, 64.0 + 2.0 ** -12]), None)
