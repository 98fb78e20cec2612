"""K9 value frames (RANGE BETWEEN) on the headline table shape: 100 M rows, key over 2^16 values (about 1 500 rows per
logical partition), an int64 "time" presort with random gaps (1 to 19, mean 10) and an f64 SUM and an f64 MAX per
frame.

Kernel figures, CUDA events, median of `--reps`: ``fb_window_range_bounds`` for ``range=(-d, 0)`` with d chosen so
that a frame holds about 7 and about 365 rows, ``fb_window_bounded`` on those bounds, and ``fb_window_frame``
(ROWS) at the same average width for comparison.  End to end: one ``fa.transform`` with a 7-day moving average
(one row per day on average).  The card's name and power limit are read in the same run.

    python tools/window_range_bench.py [--rows N] [--reps R] [--out FILE]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from fugue_b200 import kernels as K  # noqa: E402
from relational_bench import _card, timeit  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    n = a.rows
    g = torch.Generator(device=dev).manual_seed(5)
    key = torch.sort(torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)).values
    off = torch.zeros((1 << 16) + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(torch.bincount(key, minlength=1 << 16), 0)
    del key
    t = torch.cumsum(torch.randint(1, 20, (n,), dtype=torch.int64, device=dev, generator=g), 0)  # ascending times
    v = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    cols = [(K.AGG_SUM_F64, v.view(torch.int64), None), (K.AGG_MAX_F64, v.view(torch.int64), None)]
    res = {"rows": n, "partitions": 1 << 16, "columns": "f64 SUM, f64 MAX", "presort": "int64, gaps 1..19",
           "card": _card(dev)}
    frames = {}
    for d in (60, 3640):
        lo, hi = K.window_range_bounds(off, t, None, K.RANGE_KEY_I64, True, -d, 0)
        width = float((hi - lo + 1).double().mean())
        w = max(1, round(width))
        ms_b = timeit(lambda: K.window_range_bounds(off, t, None, K.RANGE_KEY_I64, True, -d, 0), reps=a.reps)
        ms_t = timeit(lambda: K.window_bounded(lo, hi, cols), reps=a.reps)
        ms_r = timeit(lambda: K.window_frame(off, n, -(w - 1), 0, cols), reps=a.reps)
        frames[str(d)] = {"mean_rows": width, "bounds_ms": ms_b, "bounded_ms": ms_t, "rows_frame_W": w,
                          "rows_frame_ms": ms_r}
        del lo, hi
    res["range_trailing"] = frames
    del off, t, v, cols
    torch.cuda.empty_cache()
    # end to end: fa.transform with a 7-day moving average
    from fugue_b200 import api as fa
    from fugue_b200.colmap import ColumnMap
    from fugue_b200.column import col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.table import B200Table

    e = fa.make_execution_engine("b200")
    g = torch.Generator(device=dev).manual_seed(4)
    days = max(1, n >> 16)  # about one row per partition and day
    T = B200DataFrame(B200Table("key:long,day:long,v0:double", [
        torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g),
        torch.randint(0, days, (n,), dtype=torch.int64, device=dev, generator=g),
        torch.randn(n, dtype=torch.float64, device=dev, generator=g)]))
    cm = ColumnMap("key", "day", "v0", f.avg(col("v0")).over(range=(-6, 0)).alias("ma7d"))
    spec = PartitionSpec(by="key", presort="day", num=256)
    ms = timeit(lambda: fa.transform(T, cm, schema="key:long,day:long,v0:double,ma7d:double", partition=spec,
                                     engine=e))
    res["transform_moving_average_7_days"] = {"ms": ms, "rows_per_s": n / ms * 1e3}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
