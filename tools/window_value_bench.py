"""FIRST_VALUE / LAST_VALUE / NTH_VALUE and NTILE / PERCENT_RANK / CUME_DIST on one H100 (DESIGN §7p, §10).

Data: ``--rows`` rows (default 100 M) in ``--parts`` logical partitions (default 65 536), sorted by (partition, an int64
presort ``t`` drawn from [0, 2^16)), a float64 value ``v`` with 5 % NULLs.  Three cases, each timed against the
composite route a user has without the new kernels, in the same process and alternating:

* (a) LAST_VALUE(v) over ``rows=(-6, 0)``: ``fb_window_value`` against torch index arithmetic (the frame's last row
  from the partition bounds) plus ``fb_gather_rows``;
* (b) NTH_VALUE(v, 2) over ``range=(-500, 0)``: ``fb_window_range_bounds`` then ``fb_window_value`` against the same
  bounds then index arithmetic plus ``fb_gather_rows``;
* (c) PERCENT_RANK + CUME_DIST + NTILE(10): ``fb_window_distribution`` against the peer bounds from ``cummax`` /
  ``cummin`` over the head bytes plus torch arithmetic.

Both routes get the partition offsets (and for (c) the peer-head bytes) as inputs.  Each time is the median of
``--runs`` CUDA-event timings after a warm-up; the outputs of the two routes are compared on every row.  The card's
name and power limit are read in the same run.

    python tools/window_value_bench.py [--rows N] [--parts P] [--runs R] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
from typing import Any, Callable, Dict, List

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from fugue_b200 import kernels as K  # noqa: E402


def card() -> Dict[str, str]:
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def timed_pair(new: Callable[[], Any], old: Callable[[], Any], runs: int) -> Dict[str, float]:
    """Median milliseconds of each route between CUDA events, alternating, after one warm-up call of each."""
    new(), old()
    torch.cuda.synchronize()
    ts: Dict[str, List[float]] = {"kernel_ms": [], "composite_ms": []}
    for _ in range(runs):
        for name, fn in (("kernel_ms", new), ("composite_ms", old)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts[name].append(a.elapsed_time(b))
    return {k: sorted(v)[len(v) // 2] for k, v in ts.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--parts", type=int, default=65_536)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("window_value_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    n = args.rows
    g = torch.Generator(device=dev).manual_seed(1)
    part = torch.randint(0, args.parts, (n,), device=dev, generator=g)
    t0 = torch.randint(0, 1 << 16, (n,), device=dev, generator=g)
    order = torch.argsort(part * (1 << 16) + t0)
    part, t = part[order], t0[order].contiguous()
    del order, t0
    v = torch.randn(n, device=dev, dtype=torch.float64, generator=g)
    m = (torch.rand(n, device=dev, generator=g) > 0.05).to(torch.uint8)
    lengths = torch.bincount(part, minlength=args.parts)
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(lengths, 0)]).contiguous()
    del part
    rows = torch.arange(n, dtype=torch.int64, device=dev)
    seg_first = torch.repeat_interleave(off[:-1], lengths, output_size=n)
    seg_last = torch.repeat_interleave(off[1:] - 1, lengths, output_size=n)
    heads = torch.ones(n, dtype=torch.uint8, device=dev)
    heads[1:] = (t[1:] != t[:-1]).to(torch.uint8)
    heads[off[:-1][lengths > 0]] = 1
    results: Dict[str, Any] = {"card": card(), "rows": n, "parts": args.parts, "runs": args.runs}

    def same(a: Any, b: Any) -> bool:
        """Equal on every row; for (value, validity) pairs the values are compared where the row is valid (the
        kernel writes 0 under a NULL, the gather the source row's bits)."""
        if len(a) == 2:
            return torch.equal(a[1], b[1]) and torch.equal(a[0][a[1] != 0], b[0][b[1] != 0])
        return all(torch.equal(x, y) for x, y in zip(a, b))

    # (a) LAST_VALUE over ROWS BETWEEN 6 PRECEDING AND CURRENT ROW
    def a_new() -> Any:
        return K.window_value(off, n, ("rows", -6, 0), [(v, m, K.VALUE_LAST)])[0]

    def a_old() -> Any:
        idx = torch.minimum(rows, seg_last)  # the frame's last row; never empty here
        (x,), (xv,) = K.gather_rows([v], [m], idx, want_valid=True)
        return x, xv

    # (b) NTH_VALUE(v, 2) over RANGE BETWEEN 500 PRECEDING AND CURRENT ROW
    def bounds() -> Any:
        return K.window_range_bounds(off, t, None, K.RANGE_KEY_I64, True, -500, 0)

    def b_new() -> Any:
        lo, hi = bounds()
        return K.window_value(off, n, ("bounds", lo, hi), [(v, m, 2)])[0]

    def b_old() -> Any:
        lo, hi = bounds()
        idx = torch.where(lo + 1 <= hi, lo + 1, torch.full_like(lo, -1))
        (x,), (xv,) = K.gather_rows([v], [m], idx, want_valid=True)
        return x, xv

    # (c) PERCENT_RANK + CUME_DIST + NTILE(10)
    def c_new() -> Any:
        pr, cd, (nt,) = K.window_distribution(off, heads, True, True, [10])
        return pr, cd, nt

    def c_old() -> Any:
        hb = heads.to(torch.bool)
        pf = torch.cummax(torch.where(hb, rows, torch.zeros_like(rows)), 0).values
        ends = torch.ones_like(hb)
        ends[:-1] = hb[1:]
        pl = torch.flip(torch.cummin(torch.flip(torch.where(ends, rows, torch.full_like(rows, n)), [0]), 0).values, [0])
        pl = torch.minimum(pl, seg_last)
        cnt = seg_last - seg_first + 1
        pr = torch.where(cnt > 1, (pf - seg_first).double() / (cnt - 1).clamp(min=1).double(), torch.zeros_like(v))
        cd = (pl - seg_first + 1).double() / cnt.double()
        r = rows - seg_first
        size = cnt // 10
        large = cnt - 10 * size
        small = large * (size + 1)
        nt = torch.where(size == 0, r + 1, torch.where(r < small, 1 + r // (size + 1),
                                                       1 + large + (r - small) // size.clamp(min=1)))
        return pr, cd, nt

    for name, new, old in (("a_last_value_rows", a_new, a_old), ("b_nth_value_range", b_new, b_old),
                           ("c_distribution", c_new, c_old)):
        res = timed_pair(new, old, args.runs)
        res["equal"] = same(new(), old())
        results[name] = res
        torch.cuda.empty_cache()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
