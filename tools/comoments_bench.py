"""Times CORR / COVAR / REGR on the device and decides their GROUP BY route (DESIGN §7k, §10).

  * ``aggregate`` of CORR(x, y) at the two shapes of the variance benchmark, 125 M rows / 10 M keys and 100 M rows /
    65 536 keys: on the hash path (the 12 pair accumulators of K6, pass A + pass B) and through
    ``_aggregate_sorted`` (key sort + co-moments scan), alternated in the same run, beside SUM and STDDEV of x;
    pass A / pass B of K6 apart (kernel times from torch.profiler, in a run of their own);
  * ``fb_segmented_comoments`` against ``fb_segmented_moments`` on one pair / one column, 100 M rows in 65 536
    segments;
  * ``fa.transform`` with a running CORR.

Algorithmic bytes come from the shapes: a co-moments scan reads x and y twice (reduce and final pass) and writes
48 bytes per row (count, two means, three sums).
Usage: python tools/comoments_bench.py [--rows-scale 1.0] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from moments_bench import DEV, card, kernel_ms, timed  # noqa: E402

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402


def table(n: int, nkeys: int) -> B200DataFrame:
    g = torch.Generator(device=DEV).manual_seed(0)
    k = torch.randint(0, nkeys, (n,), device=DEV, generator=g)
    x = torch.randn(n, device=DEV, generator=g, dtype=torch.float64) * 3 + 100
    y = x * 0.5 + torch.randn(n, device=DEV, generator=g, dtype=torch.float64)
    return B200DataFrame(B200Table("key:long,x:double,y:double", [k, x, y]))


def groupby_shapes(e, scale: float) -> list:
    out = []
    for n, nkeys in ((int(125_000_000 * scale), int(10_000_000 * scale)), (int(100_000_000 * scale), 65_536)):
        df = table(n, nkeys)
        spec = PartitionSpec(by=["key"])
        corr = [f.corr(col("x"), col("y")).alias("r")]
        row = {"rows": n, "keys": nkeys}
        row["sum_ms"] = timed(lambda: e.aggregate(df, spec, [f.sum(col("x")).alias("r")]))
        row["stddev_ms"] = timed(lambda: e.aggregate(df, spec, [f.stddev(col("x")).alias("r")]))
        # the two routes alternated, three rounds each, after one warm-up of both
        hash_ms, sorted_ms = [], []
        e._aggregate_named(df, spec, corr)
        e._aggregate_sorted(df, spec, corr)
        for _ in range(3):
            hash_ms.append(timed(lambda: e._aggregate_named(df, spec, corr), reps=1, warmup=0))
            sorted_ms.append(timed(lambda: e._aggregate_sorted(df, spec, corr), reps=1, warmup=0))
        row["corr_hash_ms"] = sorted(hash_ms)[1]
        row["corr_sorted_ms"] = sorted(sorted_ms)[1]
        row["corr_hash_all_ms"], row["corr_sorted_all_ms"] = hash_ms, sorted_ms
        row["corr_ms"] = timed(lambda: e.aggregate(df, spec, corr), reps=3)  # the route the engine takes
        ks = kernel_ms(lambda: e._aggregate_named(df, spec, corr),
                       ["fb_groupby_lean_kernel", "fb_groupby_kernel", "fb_groupby_dev_kernel", "fb_groupby_init",
                        "fb_groupby_extract"])
        row["pass_a_ms"] = ks["fb_groupby_lean_kernel"] + ks["fb_groupby_kernel"]
        row["pass_b_ms"] = ks["fb_groupby_dev_kernel"]
        row["kernels_ms"] = ks
        out.append(row)
        print(json.dumps(row), flush=True)
        del df
        torch.cuda.empty_cache()
    return out


def scan_shape(scale: float) -> dict:
    n, nseg = int(100_000_000 * scale), 65_536
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(n, device=DEV, generator=g, dtype=torch.float64)
    y = torch.randn(n, device=DEV, generator=g, dtype=torch.float64)
    off = torch.sort(torch.randint(0, n + 1, (nseg - 1,), device=DEV, generator=g)).values
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device=DEV), off,
                     torch.full((1,), n, dtype=torch.int64, device=DEV)]).contiguous()
    row = {"rows": n, "segments": nseg, "bytes": 16 * n * 2 + 48 * n}
    row["comoments_ms"] = timed(lambda: K.segmented_comoments(off, n, [(x, None, y, None)]), reps=10)
    row["moments_ms"] = timed(lambda: K.segmented_moments(off, n, [(x, None)]), reps=10)
    row["comoments_gbs"] = row["bytes"] / (row["comoments_ms"] * 1e-3) / 1e9
    print(json.dumps(row), flush=True)
    return row


def transform_shape(e, scale: float) -> dict:
    n, nkeys = int(20_000_000 * scale), 65_536
    g = torch.Generator(device=DEV).manual_seed(2)
    t = B200Table("rid:long,key:long,t:long,x:double,y:double",
                  [torch.arange(n, device=DEV), torch.randint(0, nkeys, (n,), device=DEV, generator=g),
                   torch.randint(0, 1 << 40, (n,), device=DEV, generator=g),
                   torch.randn(n, device=DEV, generator=g, dtype=torch.float64),
                   torch.randn(n, device=DEV, generator=g, dtype=torch.float64)])
    spec = PartitionSpec(by="key", presort="t")

    def run(cm):
        fa.transform(B200DataFrame(t), cm, schema="rid:long,s:double", partition=spec, engine=e, as_fugue=True)

    cc = ColumnMap("rid", f.corr(col("x"), col("y")).over(running=True).alias("s"))
    cs = ColumnMap("rid", f.stddev(col("x")).over(running=True).alias("s"))
    row = {"rows": n, "keys": nkeys, "running_corr_ms": timed(lambda: run(cc), reps=3),
           "running_stddev_ms": timed(lambda: run(cs), reps=3)}
    print(json.dumps(row), flush=True)
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows-scale", type=float, default=1.0)
    ap.add_argument("--out", default="", help="also write the whole result as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "comoments_bench measures the GPU; there is no CPU path"
    e = fa.make_execution_engine("b200")
    res = {"card": card(), "started": time.strftime("%Y-%m-%d %H:%M:%S")}
    print(json.dumps(res["card"]), flush=True)
    res["groupby"] = groupby_shapes(e, args.rows_scale)
    res["scan"] = scan_shape(args.rows_scale)
    res["transform"] = transform_shape(e, args.rows_scale)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
