"""Exact running moments, co-moments and shape moments of dyadic data, fast enough for millions of rows: the
reference of the statistics scans (``fb_segmented_moments``, ``fb_segmented_comoments``,
``fb_segmented_shape_moments``) and of the window maps built on them.

Every valid finite value is x = k / 2^10 + c with an integer k and a dyadic shift c.  The shift makes the kernel
face real cancellation, but no central sum depends on it, so the reference works on k alone: per segment and row it
keeps inclusive prefix sums S_p of k^p (and S_xy of k_x k_y) over the valid rows, built with one ``np.cumsum`` per
power minus the sum before each segment's first row.  With |k| < 2^19 for moments and co-moments (powers up to 2) and
|k| < 2^9 for shape moments (powers up to 4), every prefix sum over up to 2^23 rows stays below 2^61 and fits in
int64; the constructors assert it.  At a checked row the central sums are formed in Python integers,

    M2  = (n S2 - S1^2) / n                                  / 2^20
    M3  = (n^2 S3 - 3 n S1 S2 + 2 S1^3) / n^2                / 2^30
    M4  = (n^3 S4 - 4 n^2 S1 S3 + 6 n S1^2 S2 - 3 S1^4) / n^3 / 2^40
    Sxy = (n Sxy - Sx Sy) / n                                / 2^20

and rounded to float64 once (Python's int / int is correctly rounded; the power of two is exact).

Rules of the kernels, in ``want``: after the first valid +-inf or NaN of a segment every central sum is NaN; a
co-moments mean is then the IEEE sum of the non-finite values seen (+inf, -inf, or NaN for a NaN or for +inf with
-inf, as ``CSt``'s combine promises); where the count is 0 every output is 0.

Bounds (``bound``) are the scan bounds the suite documents, evaluated without a loop over a row's values:
  * M2: 4 m u sqrt(sum x^2 M2) (``test_moments_gpu.m2_tol(scan=True)``), sum x^2 from the integer sums exactly up
    to one float rounding;
  * co-moments: the ``errors(scan=True)`` terms of ``test_comoments_gpu``, X the running max |x| of the segment;
  * shape moments: ``oracle.shape_moments.scan_bound`` with B_2 = M2 and B_4 = M4, B_3 <= sqrt(B_2 B_4) and
    B_1 <= sqrt(m B_2) (Cauchy-Schwarz), X the running max |x|.
"""
import math
from fractions import Fraction
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np

from oracle import shape_moments as OS

U = 2.0 ** -53
BITS = 10
SCALE = 1 << BITS
MOMENT_SHIFT = 2.0 ** 20  # the shift c of moments and co-moments data
MOMENT_K = 1 << 19        # |k| < MOMENT_K for moments and co-moments
SHAPE_SHIFT = 2.0 ** 6    # the scan bound's k X B_(k-1) term would swamp M3 and M4 at a shift of 2^20
SHAPE_K = 1 << 9          # |k| < SHAPE_K for shape moments
_I64 = 2 ** 63 - 1


def dyadic(k: np.ndarray, shift: float) -> np.ndarray:
    """x = k / 2^10 + shift, exactly."""
    return np.asarray(k, dtype=np.int64) / SCALE + shift


class _Segments:
    """Segments [offsets[s], offsets[s + 1]) of n rows, and the segment id of every row."""

    def __init__(self, offsets: Any, n: int):
        self.off = np.asarray(offsets, dtype=np.int64)
        assert self.off[0] == 0 and self.off[-1] == n and np.all(np.diff(self.off) >= 0)
        self.lens = np.diff(self.off)
        self.seg = np.repeat(np.arange(len(self.lens), dtype=np.int64), self.lens)


def _running(sg: _Segments, v: np.ndarray) -> np.ndarray:
    """Inclusive prefix sums of int64 ``v`` restarting at every segment."""
    cs = np.concatenate([np.zeros(1, np.int64), np.cumsum(v, dtype=np.int64)])
    return cs[1:] - np.repeat(cs[sg.off[:-1]], sg.lens)


def _running_max(seg: np.ndarray, a: np.ndarray) -> np.ndarray:
    """Inclusive running max of int64 ``a`` in [0, 2^32) restarting at every segment."""
    assert len(a) == 0 or (a.min() >= 0 and a.max() < 1 << 32)
    key = (seg << 32) | a
    return np.maximum.accumulate(key) - (seg << 32) if len(a) else a


def _ints(a: np.ndarray) -> np.ndarray:
    """int64 array as an object array of Python ints."""
    return np.asarray(a, dtype=np.int64).astype(object)


def _round(num: np.ndarray, den: np.ndarray, bits: int) -> np.ndarray:
    """float64 of num / (den 2^bits), rounded once (object arrays of Python ints, den > 0)."""
    return (num / den).astype(np.float64) * 2.0 ** -bits


class _Column:
    """One input column over the rows that count (``rows``): its integer k, the running sums of k^p, the running
    max of |x| (in units of 2^-10), and the running counts of NaN, +inf and -inf among those rows."""

    def __init__(self, sg: _Segments, x: np.ndarray, rows: np.ndarray, shift: float, kmax: int,
                 powers: Sequence[int]):
        assert x.dtype == np.float64 and (shift * SCALE).is_integer()
        self.shift, self.c = shift, int(shift * SCALE)
        self.fin = rows & np.isfinite(x)
        k = np.where(self.fin, (x - shift) * SCALE, 0.0)
        assert np.all(np.abs(k) < kmax), "|k| too large for exact int64 sums"
        self.k = k.astype(np.int64)
        assert np.array_equal(dyadic(self.k[self.fin], shift), x[self.fin]), "values are not k / 2^10 + shift"
        assert len(x) * kmax ** max(powers) <= _I64, "prefix sums would overflow int64"
        self.s = {p: _running(sg, self.k ** p) for p in powers}
        self.amax = _running_max(sg.seg, np.where(self.fin, np.abs(self.k + self.c), 0))
        none = np.zeros(len(x), np.int64)
        self.nan, self.pinf, self.ninf = (_running(sg, (rows & f(x)).astype(np.int64)) if np.any(rows & f(x)) else none
                                          for f in (np.isnan, np.isposinf, np.isneginf))

    def bad(self) -> np.ndarray:
        return (self.nan + self.pinf + self.ninf) > 0

    def sum_sq(self, n: np.ndarray, r: np.ndarray) -> np.ndarray:
        """sum x^2 over the finite counted rows up to rows r: S2 / 2^20 + 2 c S1 / 2^10 + n c^2."""
        return (self.s[2][r] * 2.0 ** (-2 * BITS) + 2 * self.shift * self.s[1][r] * 2.0 ** -BITS
                + n[r] * self.shift ** 2)

    def mean(self, n: np.ndarray, r: np.ndarray) -> np.ndarray:
        """The mean over the counted rows up to rows r: exact and rounded once, or the IEEE sum's NaN / +-inf."""
        ok = n[r] > 0
        out = np.zeros(len(r))
        num, den = _ints(self.s[1][r][ok]) + _ints(n[r][ok]) * self.c, _ints(n[r][ok])
        out[ok] = _round(num, den, BITS)
        nan, pi, ni = self.nan[r] > 0, self.pinf[r] > 0, self.ninf[r] > 0
        out[pi] = math.inf
        out[ni] = -math.inf
        out[nan | (pi & ni)] = math.nan
        return out


class _Scan:
    count: np.ndarray  # running count of the rows that count, exact
    bad: np.ndarray    # a non-finite value among them

    def _fill(self, r: np.ndarray, vals: List[np.ndarray], bounds: List[np.ndarray], nan_words: Sequence[int]
              ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """Zero words and bounds where the count is 0; where bad, NaN words and zero bounds for ``nan_words``."""
        empty, bad = self.count[r] == 0, self.bad[r]
        for i, (v, b) in enumerate(zip(vals, bounds)):
            v[empty] = 0.0
            b[empty] = 0.0
            if i in nan_words:
                v[bad] = math.nan
                b[bad] = 0.0
        return vals, bounds


class RunningMoments(_Scan):
    """What ``K.segmented_moments`` returns for one column: per row (count, M2)."""

    def __init__(self, offsets: Any, x: np.ndarray, valid: Optional[np.ndarray], shift: float = MOMENT_SHIFT):
        n = len(x)
        sg = _Segments(offsets, n)
        ok = np.ones(n, bool) if valid is None else np.asarray(valid).astype(bool)
        self.x = _Column(sg, np.asarray(x, np.float64), ok, shift, MOMENT_K, (1, 2))
        self.count = _running(sg, ok.astype(np.int64))
        self.bad = self.x.bad()

    def m2(self, r: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """(numerator, denominator) of M2 2^20 at rows r with a finite, non-empty prefix."""
        n, s1, s2 = _ints(self.count[r]), _ints(self.x.s[1][r]), _ints(self.x.s[2][r])
        return n * s2 - s1 * s1, n

    def want(self, r: np.ndarray) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """([M2], [its bound]) at rows r."""
        r = np.asarray(r, dtype=np.int64)
        sel = (self.count[r] > 0) & ~self.bad[r]
        live = r[sel]
        m2, b = np.zeros(len(r)), np.zeros(len(r))
        m2[sel] = _round(*self.m2(live), 2 * BITS)
        b[sel] = 4 * self.count[live] * U * np.sqrt(self.x.sum_sq(self.count, live) * m2[sel])
        return self._fill(r, [m2], [b], (0,))

    def m2_fraction(self, row: int) -> Fraction:
        """The exact M2 at ``row`` (a finite, non-empty prefix)."""
        num, den = self.m2(np.array([row]))
        return Fraction(int(num[0]), int(den[0]) << (2 * BITS))


class RunningCoMoments(_Scan):
    """What ``K.segmented_comoments`` returns for one pair: per row (count, mean x, mean y, Sxx, Syy, Sxy) over the
    pair rows, where x and y are both valid."""

    def __init__(self, offsets: Any, x: np.ndarray, xvalid: Optional[np.ndarray], y: np.ndarray,
                 yvalid: Optional[np.ndarray], shift_x: float = MOMENT_SHIFT, shift_y: float = MOMENT_SHIFT):
        n = len(x)
        sg = _Segments(offsets, n)
        ok = np.ones(n, bool)
        for v in (xvalid, yvalid):
            if v is not None:
                ok &= np.asarray(v).astype(bool)
        self.x = _Column(sg, np.asarray(x, np.float64), ok, shift_x, MOMENT_K, (1, 2))
        self.y = _Column(sg, np.asarray(y, np.float64), ok, shift_y, MOMENT_K, (1, 2))
        assert n * MOMENT_K ** 2 <= _I64
        self.sxy = _running(sg, self.x.k * self.y.k)
        self.count = _running(sg, ok.astype(np.int64))
        self.bad = self.x.bad() | self.y.bad()

    def sums(self, r: np.ndarray) -> Tuple[Tuple[np.ndarray, ...], np.ndarray]:
        """((numerators of Sxx, Syy, Sxy) 2^20, denominator) at rows r with a finite, non-empty prefix."""
        n = _ints(self.count[r])
        sx, sy = _ints(self.x.s[1][r]), _ints(self.y.s[1][r])
        return (n * _ints(self.x.s[2][r]) - sx * sx, n * _ints(self.y.s[2][r]) - sy * sy,
                n * _ints(self.sxy[r]) - sx * sy), n

    def want(self, r: np.ndarray) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """([mean x, mean y, Sxx, Syy, Sxy], [their bounds]) at rows r."""
        r = np.asarray(r, dtype=np.int64)
        sel = (self.count[r] > 0) & ~self.bad[r]
        live = r[sel]
        vals = [self.x.mean(self.count, r), self.y.mean(self.count, r)] + [np.zeros(len(r)) for _ in range(3)]
        nums, den = self.sums(live)
        for i, num in enumerate(nums):
            vals[2 + i][sel] = _round(num, den, 2 * BITS)
        m = self.count[live].astype(np.float64)
        nx, ny = np.sqrt(self.x.sum_sq(self.count, live)), np.sqrt(self.y.sum_sq(self.count, live))
        ax, ay = self.x.amax[live] / SCALE, self.y.amax[live] / SCALE
        sxx, syy = vals[2][sel], vals[3][sel]
        terms = (ax, ay, nx * np.sqrt(sxx), ny * np.sqrt(syy), np.maximum(nx * np.sqrt(syy), ny * np.sqrt(sxx)))
        bounds = [np.zeros(len(r)) for _ in range(5)]
        for b, t in zip(bounds, terms):
            b[sel] = 4 * m * U * t
        # where bad, a mean whose column had no non-finite value is still exact and within its bound
        for i, c in enumerate((self.x, self.y)):
            fin = (self.count[r] > 0) & self.bad[r] & ~c.bad()[r]
            bounds[i][fin] = 4 * self.count[r][fin] * U * c.amax[r][fin] / SCALE
        return self._fill(r, vals, bounds, (2, 3, 4))

    def state(self, row: int) -> Tuple:
        """The exact state at ``row`` in the form of ``oracle.comoments.exact_state`` (a finite prefix)."""
        r = np.array([row])
        m = int(self.count[row])
        if m == 0:
            return 0, None, None, None, None, None
        nums, den = self.sums(r)
        means = [Fraction(int(c.s[1][row]) + m * c.c, m * SCALE) for c in (self.x, self.y)]
        return (m, *means, *(Fraction(int(q[0]), m << (2 * BITS)) for q in nums))

    def errors(self, row: int) -> Tuple[float, ...]:
        """The bounds of ``state(row)``'s words, as ``test_comoments_gpu.errors(scan=True)`` gives them."""
        return tuple(float(b[0]) for b in self.want(np.array([row]))[1])


class RunningShapeMoments(_Scan):
    """What ``K.segmented_shape_moments`` returns for one column: per row (count, M2, M3, M4)."""

    def __init__(self, offsets: Any, x: np.ndarray, valid: Optional[np.ndarray], shift: float = SHAPE_SHIFT):
        n = len(x)
        sg = _Segments(offsets, n)
        ok = np.ones(n, bool) if valid is None else np.asarray(valid).astype(bool)
        self.x = _Column(sg, np.asarray(x, np.float64), ok, shift, SHAPE_K, (1, 2, 3, 4))
        self.count = _running(sg, ok.astype(np.int64))
        self.bad = self.x.bad()

    def sums(self, r: np.ndarray) -> Tuple[Tuple[np.ndarray, ...], Tuple[np.ndarray, ...]]:
        """((numerators of M2 2^20, M3 2^30, M4 2^40), (their denominators)) at rows r with a finite, non-empty
        prefix."""
        n = _ints(self.count[r])
        s1, s2, s3, s4 = (_ints(self.x.s[p][r]) for p in (1, 2, 3, 4))
        return ((n * s2 - s1 * s1, n * n * s3 - 3 * n * s1 * s2 + 2 * s1 ** 3,
                 n ** 3 * s4 - 4 * n * n * s1 * s3 + 6 * n * s1 * s1 * s2 - 3 * s1 ** 4), (n, n * n, n ** 3))

    def want(self, r: np.ndarray) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """([M2, M3, M4], [their bounds]) at rows r."""
        r = np.asarray(r, dtype=np.int64)
        sel = (self.count[r] > 0) & ~self.bad[r]
        live = r[sel]
        vals = [np.zeros(len(r)) for _ in range(3)]
        nums, dens = self.sums(live)
        for i, (num, den) in enumerate(zip(nums, dens)):
            vals[i][sel] = _round(num, den, (i + 2) * BITS)
        m = self.count[live].astype(np.float64)
        m2, m4 = vals[0][sel], vals[2][sel]
        b = (np.sqrt(m * m2), m2, np.sqrt(m2 * m4), m4)
        bounds = [np.zeros(len(r)) for _ in range(3)]
        for out, d in zip(bounds, OS.scan_bound(m, self.x.amax[live] / SCALE, b)):
            out[sel] = d
        return self._fill(r, vals, bounds, (0, 1, 2))

    def central_sums(self, row: int) -> OS.Moments:
        """The exact (m, M2, M3, M4) at ``row``, as ``oracle.shape_moments.central_sums`` gives them."""
        m = int(self.count[row])
        if m == 0 or self.bad[row]:
            return m, None, None, None
        nums, dens = self.sums(np.array([row]))
        return (m, *(Fraction(int(q[0]), int(d[0]) << (k * BITS)) for k, q, d in zip((2, 3, 4), nums, dens)))

    def bounds(self, row: int) -> Tuple[float, ...]:
        """The bounds on the computed M2, M3, M4 at ``row``."""
        return tuple(float(b[0]) for b in self.want(np.array([row]))[1])
