"""K9 moving frames (ROWS BETWEEN) on the headline table shape: 100 M rows, key over 2^16 values (about 1 500
rows per logical partition), an f64 SUM and an f64 MAX per frame.

Kernel figures: ``fb_window_frame`` for trailing frames of width W (both paths: W up to FRAME_TILE_MAX_WIDTH
runs in one pass, wider frames on the scan path) beside ``fb_segmented_scan`` on the same two columns, CUDA
events, median of `--reps`.  Algorithmic bytes: read the 8-byte value, write value and count, 24 B per row and
column.  End to end: one ``fa.transform`` with a 7-row moving average.  The card's name and power limit are
read in the same run.

    python tools/window_frame_bench.py [--rows N] [--reps R] [--out FILE]
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
    v = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    cols = [(K.AGG_SUM_F64, v.view(torch.int64), None), (K.AGG_MAX_F64, v.view(torch.int64), None)]
    alg = len(cols) * n * 24
    tw = K.FRAME_TILE_MAX_WIDTH
    res = {"rows": n, "partitions": 1 << 16, "columns": "f64 SUM, f64 MAX", "card": _card(dev)}
    ms_scan = timeit(lambda: K.segmented_scan(off, n, cols), reps=a.reps)
    res["segmented_scan"] = {"ms": ms_scan, "alg_TBps": alg / ms_scan / 1e9}
    frames = {}
    for w in [3, 7, 30, 365, tw, tw + 1]:
        ms = timeit(lambda: K.window_frame(off, n, -(w - 1), 0, cols), reps=a.reps)
        frames[str(w)] = {"path": "one pass" if w <= tw else "scan", "ms": ms, "alg_TBps": alg / ms / 1e9,
                          "vs_scan": ms_scan / ms}
    res["window_frame_trailing"] = frames
    del key, off, v, cols
    torch.cuda.empty_cache()
    # end to end: fa.transform with a 7-row moving average
    from fugue_b200 import api as fa
    from fugue_b200.colmap import ColumnMap
    from fugue_b200.column import col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.table import B200Table

    e = fa.make_execution_engine("b200")
    g = torch.Generator(device=dev).manual_seed(4)
    T = B200DataFrame(B200Table("key:long,i1:long,v0:double", [
        torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g),
        torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g),
        torch.randn(n, dtype=torch.float64, device=dev, generator=g)]))
    cm = ColumnMap("key", "i1", "v0", f.avg(col("v0")).over(rows=(-6, 0)).alias("ma7"))
    spec = PartitionSpec(by="key", presort="i1", num=256)
    ms = timeit(lambda: fa.transform(T, cm, schema="key:long,i1:long,v0:double,ma7:double", partition=spec, engine=e))
    res["transform_moving_average_7"] = {"ms": ms, "rows_per_s": n / ms * 1e3}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
