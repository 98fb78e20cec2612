"""Times the exponentially weighted window functions on the device (DESIGN §7s, §10).

  * ``ewm_mean`` and ``ewm_std`` of one float64 column through the window evaluation of a ColumnMap (``_with_windows``
    over logical partitions), beside ``avg(...).over(running=True)`` and ``stddev(...).over(running=True)`` through the
    same path, at 100 M rows in 65 536 partitions and in one;
  * the scans alone: ``fb_segmented_ewm`` writing the count and mean (what ``ewm_mean`` reads) and writing W, W2 and C
    as well (what ``ewm_std`` reads), against ``fb_segmented_moments`` on the same column;
  * pandas ``groupby().ewm().mean()`` on a 1 M-row slice in 65 536 groups, the host-callback baseline.

Algorithmic bytes come from the shapes: a scan reads the 8-byte values twice (reduce and final pass) and writes 8 bytes
per row for the count and for each output (one for the moments scan, one or four for the ewm scan).  The card's name,
power limit and clocks are read in the same run.  Prints one JSON line per shape and one for the whole run; writes a
file only when given ``--out``.
Usage: python tools/ewm_bench.py [--rows-scale 1.0] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fugue_b200 import colmap  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402
from moments_bench import card, timed  # noqa: E402

DEV = torch.device("cuda", 0)


def offsets(n: int, nseg: int, g: torch.Generator) -> torch.Tensor:
    cut = torch.sort(torch.randint(0, n + 1, (nseg - 1,), device=DEV, generator=g)).values
    return torch.cat([torch.zeros(1, dtype=torch.int64, device=DEV), cut,
                      torch.full((1,), n, dtype=torch.int64, device=DEV)]).contiguous()


def shape(n: int, nseg: int) -> dict:
    g = torch.Generator(device=DEV).manual_seed(1)
    v = torch.randn(n, device=DEV, generator=g, dtype=torch.float64) * 3 + 100
    off = offsets(n, nseg, g)
    t = B200Table("v:double", [v])
    t.logical_offsets = off
    t.logical_order = []
    nodes = {"ewm_mean": f.ewm_mean(col("v"), alpha=0.1), "ewm_std": f.ewm_std(col("v"), alpha=0.1),
             "avg_running": f.avg(col("v")).over(running=True), "stddev_running": f.stddev(col("v")).over(running=True)}
    row = {"rows": n, "segments": nseg, "moments_scan_bytes": 8 * n * 2 + 16 * n, "ewm_scan_bytes": 8 * n * 2 + 16 * n,
           "ewm_scan_spread_bytes": 8 * n * 2 + 40 * n}
    for name, e in nodes.items():
        row[f"{name}_ms"] = timed(lambda e=e: colmap._with_windows(t, [e.alias("r")]), reps=10)
    for name, spread in (("ewm_scan", False), ("ewm_scan_spread", True)):
        row[f"{name}_ms"] = timed(lambda spread=spread: K.segmented_ewm(
            off, n, [(v, None, 0.1, True, K.EWM_ROWS, None, 1.0, spread)]), reps=10)
        row[f"{name}_gbs"] = row[f"{name}_bytes"] / (row[f"{name}_ms"] * 1e-3) / 1e9
    row["moments_scan_ms"] = timed(lambda: K.segmented_moments(off, n, [(v, None)]), reps=10)
    row["moments_scan_gbs"] = row["moments_scan_bytes"] / (row["moments_scan_ms"] * 1e-3) / 1e9
    print(json.dumps(row), flush=True)
    return row


def pandas_slice(n: int = 1_000_000, nseg: int = 65_536) -> dict:
    import pandas as pd

    rng = np.random.default_rng(1)
    df = pd.DataFrame({"k": np.sort(rng.integers(0, nseg, n)), "v": rng.normal(100, 3, n)})
    t0 = time.perf_counter()
    df.groupby("k")["v"].ewm(alpha=0.1).mean()
    row = {"pandas_rows": n, "pandas_groups": nseg, "pandas_groupby_ewm_mean_ms": (time.perf_counter() - t0) * 1e3}
    print(json.dumps(row), flush=True)
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows-scale", type=float, default=1.0)
    ap.add_argument("--out", default="", help="also write the whole result as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ewm_bench measures the GPU; there is no CPU path"
    res = {"card": card(), "started": time.strftime("%Y-%m-%d %H:%M:%S")}
    print(json.dumps(res["card"]), flush=True)
    n = int(100_000_000 * args.rows_scale)
    res["shapes"] = [shape(n, 65_536), shape(n, 1)]
    res["pandas"] = pandas_slice()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
