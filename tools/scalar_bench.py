"""CASE, % and the numeric functions in the expression evaluator (K8) at 100 M rows, and the 3-expression SELECT of
tools/relational_bench.py as a regression check.  Prints one JSON object; the card name and its power limit are read
in the same run.

    python tools/scalar_bench.py [--tree DIR]   # DIR: another checkout to import instead (e.g. a parent build)
    python tools/scalar_bench.py --select-only   # only the regression SELECT
"""
import argparse
import json
import os
import subprocess
import sys


def timeit(fn, reps=7):
    import torch

    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def card() -> dict:
    import torch

    out = {"device": torch.cuda.get_device_name(0)}
    try:  # a read-only query
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--select-only", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch

    from fugue_b200 import api as fa
    from fugue_b200.column import SelectColumns, col
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    e = fa.make_execution_engine("b200")
    n = 100_000_000
    key = torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)
    v0 = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    v1 = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    T = B200DataFrame(B200Table("key:long,v0:double,v1:double", [key, v0, v1]))
    out = card()
    sel = SelectColumns((col("v0") * col("v1") + col("key")).alias("x"), ((col("v0") > 0) & (col("v1") < 0.5)).alias("p"),
                        (col("key") * 3 - 7).alias("k3"))
    ms = timeit(lambda: e.select(T, sel))
    out["select_3_exprs"] = {"rows": n, "ms": ms, "alg_GBps": 41 * n / ms / 1e6}
    if not args.select_only:
        from fugue_b200.column import functions as ff

        vi = torch.randint(-(1 << 40), 1 << 40, (n,), dtype=torch.int64, device=dev, generator=g)
        TI = B200DataFrame(B200Table("v0:long", [vi]))
        work = {
            "case_when": (T, (ff.case([(col("v0") > 0, col("v1"))], -col("v1"))).alias("r"), 24),
            "mod_int64": (TI, (col("v0") % 7).alias("r"), 16),
            "sqrt_abs_plus_round": (T, (ff.sqrt(ff.abs(col("v0"))) + ff.round(col("v1"), 2)).alias("r"), 24),
            "power_2": (T, ff.power(col("v0"), 2).alias("r"), 16 + 1),  # + the validity byte (a domain error is NULL)
        }
        for name, (tab, expr, bytes_per_row) in work.items():
            ms = timeit(lambda: e.select(tab, SelectColumns(expr)))
            out[name] = {"rows": n, "ms": ms, "alg_GBps": bytes_per_row * n / ms / 1e6, "bytes_per_row": bytes_per_row}
        K = B200DataFrame(B200Table("key:long,v0:double,v1:double", [key % 1024, v0, v1]))
        agg = [ff.sum(ff.case([(col("v0") > 0, col("v1"))], 0.0)).alias("s")]
        ms = timeit(lambda: e.aggregate(K, PartitionSpec(by=["key"]), agg))
        out["sum_case_group_by"] = {"rows": n, "groups": 1024, "ms": ms, "alg_GBps": 24 * n / ms / 1e6}
        base = [ff.sum(col("v1")).alias("s")]
        ms = timeit(lambda: e.aggregate(e.filter(K, col("v0") > 0), PartitionSpec(by=["key"]), base))
        out["filter_then_sum_group_by"] = {"rows": n, "groups": 1024, "ms": ms}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
