"""Times the shape statistics on the device (DESIGN §7m, §10).

  * ``fa.aggregate`` SUM, STDDEV, SKEWNESS and KURTOSIS on the hash path at 125 M rows / 10 M keys and 100 M rows /
    65 536 keys, KURTOSIS through ``_aggregate_sorted`` (key sort + shape-moments scan), and pass A / pass B of K6
    apart for STDDEV, SKEWNESS and KURTOSIS (kernel times from torch.profiler, in runs of their own);
  * ``fb_segmented_shape_moments`` against ``fb_segmented_moments`` on one f64 column, 100 M rows in 65 536 segments.

Algorithmic bytes come from the shapes: a group-by pass reads the 8-byte key and the 8-byte value of every row; a
scan reads the values twice (reduce and final pass) and writes 8 bytes per row for the count and for each output.
The card's name, power limit and clocks are read in the same run.  Prints one JSON line per shape and one for the
whole run; writes a file only when given ``--out``.
Usage: python tools/shape_moments_bench.py [--rows-scale 1.0] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from moments_bench import card, kernel_ms, table, timed  # noqa: E402

DEV = torch.device("cuda", 0)
KERNELS = ["fb_groupby_lean_kernel", "fb_groupby_kernel", "fb_groupby_dev_kernel", "fb_groupby_init",
           "fb_groupby_extract"]


def groupby_shapes(e, scale: float) -> list:
    out = []
    for n, nkeys in ((int(125_000_000 * scale), int(10_000_000 * scale)), (int(100_000_000 * scale), 65_536)):
        df = table(n, nkeys)
        spec = PartitionSpec(by=["key"])
        row = {"rows": n, "keys": nkeys, "bytes_per_pass": 16 * n}
        aggs = (("sum", f.sum(col("v"))), ("stddev", f.stddev(col("v"))), ("skewness", f.skewness(col("v"))),
                ("kurtosis", f.kurtosis(col("v"))))
        for name, a in aggs:
            row[f"{name}_ms"] = timed(lambda a=a: e.aggregate(df, spec, [a.alias("r")]))
        row["kurtosis_sorted_ms"] = timed(lambda: e._aggregate_sorted(df, spec, [f.kurtosis(col("v")).alias("r")]),
                                          reps=3)
        for name, a in aggs[1:]:
            ks = kernel_ms(lambda a=a: e.aggregate(df, spec, [a.alias("r")]), KERNELS)
            row[f"{name}_pass_a_ms"] = ks["fb_groupby_lean_kernel"] + ks["fb_groupby_kernel"]
            row[f"{name}_pass_b_ms"] = ks["fb_groupby_dev_kernel"]
        out.append(row)
        print(json.dumps(row), flush=True)
        del df
        torch.cuda.empty_cache()
    return out


def scan_shape(scale: float) -> dict:
    n, nseg = int(100_000_000 * scale), 65_536
    g = torch.Generator(device=DEV).manual_seed(1)
    v = torch.randn(n, device=DEV, generator=g, dtype=torch.float64)
    off = torch.sort(torch.randint(0, n + 1, (nseg - 1,), device=DEV, generator=g)).values
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device=DEV), off,
                     torch.full((1,), n, dtype=torch.int64, device=DEV)]).contiguous()
    row = {"rows": n, "segments": nseg, "moments_bytes": 8 * n * 2 + 16 * n, "shape_bytes": 8 * n * 2 + 32 * n}
    row["moments_ms"] = timed(lambda: K.segmented_moments(off, n, [(v, None)]), reps=10)
    row["shape_moments_ms"] = timed(lambda: K.segmented_shape_moments(off, n, [(v, None)]), reps=10)
    row["moments_gbs"] = row["moments_bytes"] / (row["moments_ms"] * 1e-3) / 1e9
    row["shape_moments_gbs"] = row["shape_bytes"] / (row["shape_moments_ms"] * 1e-3) / 1e9
    print(json.dumps(row), flush=True)
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows-scale", type=float, default=1.0)
    ap.add_argument("--out", default="", help="also write the whole result as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "shape_moments_bench measures the GPU; there is no CPU path"
    e = fa.make_execution_engine("b200")
    res = {"card": card(), "started": time.strftime("%Y-%m-%d %H:%M:%S")}
    print(json.dumps(res["card"]), flush=True)
    res["groupby"] = groupby_shapes(e, args.rows_scale)
    res["scan"] = scan_shape(args.rows_scale)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
