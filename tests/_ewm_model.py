"""A float64 model of the ``EwSt`` state of ``fb_segmented_ewm`` (csrc/fb_window.cu, DESIGN §7s): the entry, the
combine and the output, written as the kernel writes them, for folding random splits of a series into runs."""
import math
from typing import List, NamedTuple, Optional, Sequence, Tuple


class Op(NamedTuple):
    k: float       # log2(beta), or -1 / halflife for times
    alpha: float
    adjust: bool
    obs: bool      # positions are observation ordinals


class St(NamedTuple):
    c: int
    t1: int
    tl: int
    x1: float
    q: float
    w: float
    w2: float
    mean: float
    cm: float
    f: bool = False


EMPTY = St(0, 0, 0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)


def make_op(alpha: float, adjust: bool, ignore_na: bool, scale: Optional[float] = None) -> Op:
    k = -scale if scale is not None else (math.log2(1.0 - alpha) if alpha < 1.0 else -math.inf)
    return Op(k, alpha, adjust, ignore_na and scale is None)


def decay(op: Op, dt: int) -> float:
    return 1.0 if dt == 0 else 2.0 ** (op.k * dt)


def merge(a: Tuple[float, ...], b: Tuple[float, ...]) -> Tuple[float, ...]:
    if a[0] == 0.0:
        return (b[0], a[1] + b[1], b[2], a[3] + b[3])
    w = a[0] + b[0]
    d = b[2] - a[2]
    wb = b[0] / w
    mean = a[2] + d * wb if math.isfinite(d) else (a[2] * a[0] + b[2] * b[0]) / w
    return (w, a[1] + b[1], mean, a[3] + b[3] + d * d * a[0] * wb)


def total(s: St) -> Tuple[float, ...]:
    p = (s.q, s.q * s.q, s.x1, s.x1 - s.x1)
    return merge(p, (s.w, s.w2, s.mean, s.cm)) if s.c > 1 else p


def combine(op: Op, a: St, b: St) -> St:
    if b.f:
        return b
    if b.c == 0:
        return a
    if a.c == 0:
        return b._replace(f=a.f)
    if op.adjust:
        fa = decay(op, b.c if op.obs else b.tl - a.tl)
        w1 = b.q
    else:
        bg = decay(op, 1 if op.obs else b.t1 - a.tl)
        den = bg + op.alpha
        fa = b.q * (bg / den)
        w1 = b.q * (op.alpha / den)
    r = (w1, w1 * w1, b.x1, b.x1 - b.x1)
    if a.c > 1:
        r = merge((a.w * fa, a.w2 * fa * fa, a.mean, a.cm * fa), r)
    if b.c > 1:
        r = merge(r, (b.w, b.w2, b.mean, b.cm))
    return St(a.c + b.c, a.t1, b.tl, a.x1, a.q * fa, *r, f=a.f)


def entry(x: Optional[float], t: int, head: bool = False) -> St:
    obs = x is not None and x == x
    return St(int(obs), t, t, x if obs else 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, head)


def fold(op: Op, xs: Sequence[Optional[float]], ts: Sequence[int], cuts: Sequence[int]) -> List[Tuple[float, ...]]:
    """Per row, (count, mean, W, W2, C) (without adjust, W, W2 and C over weight shares: W = 1) of the series cut into runs at ``cuts``: each run is folded alone, then the
    prefix of the earlier runs is combined with the run's prefix at every row, as pass 3 does."""
    out: List[Tuple[float, ...]] = []
    bounds = [0] + sorted(set(c for c in cuts if 0 < c < len(xs))) + [len(xs)]
    carry = EMPTY
    for lo, hi in zip(bounds, bounds[1:]):
        run = EMPTY
        for i in range(lo, hi):
            run = combine(op, run, entry(xs[i], ts[i], i == 0))
            s = combine(op, carry, run)
            out.append((s.c,) + ((0.0,) * 4 if s.c == 0 else tuple(total(s)[j] for j in (2, 0, 1, 3))))
        carry = combine(op, carry, run)
    return out
