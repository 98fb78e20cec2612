"""Date and timestamp expressions in the expression evaluator (K8) at 100 M ``timestamp[us]`` rows, and the 3-expression
SELECT of tools/relational_bench.py as a regression check.  Prints one JSON object; the card name and its power limit
are read in the same run.  Times are medians of CUDA-event timings after a warm-up call.

    python tools/temporal_bench.py
    python tools/temporal_bench.py --select-only [--tree DIR]   # only the regression SELECT; DIR: another checkout to
                                                                 # import instead (e.g. a build of the parent commit)
"""
import argparse
import datetime
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from scalar_bench import card, timeit  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--select-only", action="store_true")
    ap.add_argument("--rows", type=int, default=100_000_000)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import pyarrow as pa
    import torch

    from fugue_b200 import api as fa
    from fugue_b200.column import SelectColumns, col
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.schema import Schema
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    e = fa.make_execution_engine("b200")
    n = args.rows
    out = card()
    out["tree"] = os.path.abspath(args.tree)
    key = torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)
    v0 = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    v1 = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    T = B200DataFrame(B200Table("key:long,v0:double,v1:double", [key, v0, v1]))
    sel = SelectColumns((col("v0") * col("v1") + col("key")).alias("x"), ((col("v0") > 0) & (col("v1") < 0.5)).alias("p"),
                        (col("key") * 3 - 7).alias("k3"))
    reps = [timeit(lambda: e.select(T, sel)) for _ in range(3)]
    out["select_3_exprs"] = {"rows": n, "ms": sorted(reps)[1], "ms_runs": reps, "alg_GBps": 41 * n / sorted(reps)[1] / 1e6}
    if args.select_only:
        print(json.dumps(out))
        return
    del T, v1
    from fugue_b200.column import functions as ff, lit

    us_day = 86_400_000_000
    lo, hi = 18_000 * us_day, 20_000 * us_day  # 2019-04 .. 2024-10
    t = torch.randint(lo, hi, (n,), dtype=torch.int64, device=dev, generator=g)
    day = torch.div(t, us_day, rounding_mode="floor")
    TS = B200DataFrame(B200Table(Schema([pa.field("t", pa.timestamp("us")), pa.field("raw", pa.int64()),
                                         pa.field("day", pa.int64()), pa.field("v", pa.float64())]), [t, t, day, v0]))
    cut = datetime.datetime(1970, 1, 1) + datetime.timedelta(days=19_400)  # keeps 30 % of the rows
    cut_raw = 19_400 * us_day

    def rate(ms, bytes_per_row):
        return {"rows": n, "ms": ms, "bytes_per_row": bytes_per_row, "alg_TBps": bytes_per_row * n / ms / 1e9,
                "share_of_3.35_TBps": bytes_per_row * n / ms / 1e9 / 3.35}

    ymd = SelectColumns(ff.year(col("t")).alias("y"), ff.month(col("t")).alias("m"), ff.day(col("t")).alias("d"))
    out["select_year_month_day"] = rate(timeit(lambda: e.select(TS, ymd)), 8 + 24)
    out["select_date_trunc_month"] = rate(timeit(lambda: e.select(TS, SelectColumns(ff.date_trunc("month", col("t")).alias("m")))), 16)
    out["select_raw_plus_1"] = rate(timeit(lambda: e.select(TS, SelectColumns((col("raw") + 1).alias("m")))), 16)
    out["filter_timestamp_literal"] = {"rows": n, "ms": timeit(lambda: e.filter(TS, col("t") >= lit(cut))),
                                       "kept": float((t >= cut_raw).float().mean())}
    out["filter_raw_int64"] = {"rows": n, "ms": timeit(lambda: e.filter(TS, col("raw") >= cut_raw))}
    agg = [ff.sum(col("v")).alias("s")]
    by_trunc = SelectColumns(ff.date_trunc("day", col("t")).alias("dd"), ff.sum(col("v")).alias("s"))
    out["group_by_date_trunc_day"] = {"rows": n, "groups": 2000, "ms": timeit(lambda: e.select(TS, by_trunc))}
    out["group_by_day_column"] = {"rows": n, "groups": 2000, "ms": timeit(lambda: e.aggregate(TS, PartitionSpec(by=["day"]), agg))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
