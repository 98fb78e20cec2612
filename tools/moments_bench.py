"""Times the variance family on the device (DESIGN §7i, §10).

  * ``fa.aggregate`` SUM, AVG and STDDEV at 125 M rows / 10 M keys and 100 M rows / 65 536 keys: STDDEV on the
    hash path (pass A + pass B of K6) and through ``_aggregate_sorted`` (key sort + moments scan), and pass A /
    pass B of K6 apart (kernel times from torch.profiler, in a run of their own);
  * ``fb_segmented_moments`` against ``fb_segmented_scan`` SUM on one f64 column, 100 M rows in 65 536 segments;
  * ``fa.transform`` with a running STDDEV.

Algorithmic bytes come from the shapes: a group-by pass reads the 8-byte key and the 8-byte value of every row;
a scan reads the values twice (reduce and final pass) and writes 16 bytes per row (count and result).
Usage: python tools/moments_bench.py [--rows-scale 1.0] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402

DEV = torch.device("cuda", 0)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [x.strip() for x in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def timed(fn, reps: int = 5, warmup: int = 1) -> float:
    """Median milliseconds of ``fn`` between CUDA events, after a device synchronise."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return sorted(out)[len(out) // 2]


def kernel_ms(fn, names) -> dict:
    """Device time per kernel-name prefix of one call of ``fn``, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    res = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                res[n] += ev.device_time_total / 1000.0
    return res


def table(n: int, nkeys: int) -> B200DataFrame:
    g = torch.Generator(device=DEV).manual_seed(0)
    k = torch.randint(0, nkeys, (n,), device=DEV, generator=g)
    v = torch.randn(n, device=DEV, generator=g, dtype=torch.float64) * 3 + 100
    return B200DataFrame(B200Table("key:long,v:double", [k, v]))


def groupby_shapes(e, scale: float) -> list:
    out = []
    for n, nkeys in ((int(125_000_000 * scale), int(10_000_000 * scale)), (int(100_000_000 * scale), 65_536)):
        df = table(n, nkeys)
        spec = PartitionSpec(by=["key"])
        row = {"rows": n, "keys": nkeys, "bytes_per_pass": 16 * n}
        for name, a in (("sum", f.sum(col("v"))), ("avg", f.avg(col("v"))), ("stddev", f.stddev(col("v")))):
            row[f"{name}_ms"] = timed(lambda a=a: e.aggregate(df, spec, [a.alias("r")]))
        row["stddev_sorted_ms"] = timed(lambda: e._aggregate_sorted(df, spec, [f.stddev(col("v")).alias("r")]),
                                        reps=3)
        ks = kernel_ms(lambda: e.aggregate(df, spec, [f.stddev(col("v")).alias("r")]),
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
    v = torch.randn(n, device=DEV, generator=g, dtype=torch.float64)
    off = torch.sort(torch.randint(0, n + 1, (nseg - 1,), device=DEV, generator=g)).values
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device=DEV), off,
                     torch.full((1,), n, dtype=torch.int64, device=DEV)]).contiguous()
    row = {"rows": n, "segments": nseg, "bytes": 8 * n * 2 + 16 * n}
    row["moments_ms"] = timed(lambda: K.segmented_moments(off, n, [(v, None)]), reps=10)
    row["scan_sum_ms"] = timed(lambda: K.segmented_scan(off, n, [(K.AGG_SUM_F64, v, None)]), reps=10)
    for k in ("moments", "scan_sum"):
        row[f"{k}_gbs"] = row["bytes"] / (row[f"{k}_ms"] * 1e-3) / 1e9
    print(json.dumps(row), flush=True)
    return row


def transform_shape(e, scale: float) -> dict:
    n, nkeys = int(20_000_000 * scale), 65_536
    g = torch.Generator(device=DEV).manual_seed(2)
    t = B200Table("rid:long,key:long,t:long,v:double",
                  [torch.arange(n, device=DEV), torch.randint(0, nkeys, (n,), device=DEV, generator=g),
                   torch.randint(0, 1 << 40, (n,), device=DEV, generator=g),
                   torch.randn(n, device=DEV, generator=g, dtype=torch.float64)])
    cm = ColumnMap("rid", f.stddev(col("v")).over(running=True).alias("s"))
    spec = PartitionSpec(by="key", presort="t")

    def run():
        fa.transform(B200DataFrame(t), cm, schema="rid:long,s:double", partition=spec, engine=e, as_fugue=True)

    cs = ColumnMap("rid", f.sum(col("v")).over(running=True).alias("s"))

    def run_sum():
        fa.transform(B200DataFrame(t), cs, schema="rid:long,s:double", partition=spec, engine=e, as_fugue=True)

    row = {"rows": n, "keys": nkeys, "running_stddev_ms": timed(run, reps=3),
           "running_sum_ms": timed(run_sum, reps=3)}
    print(json.dumps(row), flush=True)
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows-scale", type=float, default=1.0)
    ap.add_argument("--out", default="", help="also write the whole result as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "moments_bench measures the GPU; there is no CPU path"
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
