"""Casts from strings (K13) at 100 M rows of int32 codes over dictionaries of 1 000 and 10 M entries of three kinds:
decimal integers, shortest-repr doubles and ISO timestamps with microseconds.  Prints one JSON object; the card name
and its power limit are read in the same run.  Times are medians of CUDA-event timings after a warm-up call.

Per dictionary: ``fb_string_parse`` alone and the entry bytes it reads per second, against pyarrow's ``cast`` of the
same dictionary on one host core; ``SELECT SUM(CAST(s AS double))`` on its first call (upload and parse included) and
on a cached call (the timestamps: MAX(CAST(s AS timestamp))).  Then ``alter_columns`` of a 10 M-row frame on the device against the host round trip the base
``DataFrame.alter_columns`` makes.

    python tools/string_cast_bench.py [--rows N]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scalar_bench import card, timeit  # noqa: E402


def dictionary(kind: str, m: int, seed: int):
    import numpy as np
    import pyarrow as pa
    import pyarrow.compute as pc

    rng = np.random.default_rng(seed)
    if kind == "int":
        return pc.cast(pa.array(rng.integers(-(1 << 40), 1 << 40, m)), pa.string()), pa.int64()
    if kind == "double":  # Arrow formats a double as its shortest round-trip decimal
        return pc.cast(pa.array(rng.standard_normal(m) * 10.0 ** rng.integers(-8, 9, m)), pa.string()), pa.float64()
    us = rng.integers(0, 2_000_000_000_000_000, m)  # 1970 .. 2033, microseconds
    return pc.cast(pa.array(us, type=pa.timestamp("us")), pa.string()), pa.timestamp("us")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    args = ap.parse_args()
    import pyarrow as pa
    import pyarrow.compute as pc
    import torch

    from fugue_b200 import api as fa
    from fugue_b200 import kernels as K
    from fugue_b200 import strings as ST
    from fugue_b200.column import SelectColumns, col, functions as ff
    from fugue_b200.dataframe import B200DataFrame, DataFrame
    from fugue_b200.schema import Schema
    from fugue_b200.table import B200Table

    pa.set_cpu_count(1)
    dev = torch.device("cuda", 0)
    e = fa.make_execution_engine("b200")
    n = args.rows
    out = card()
    out["rows"] = n
    runs = []
    for kind in ("int", "double", "timestamp"):
        for m in (1000, 10_000_000):
            d, tp = dictionary(kind, m, m)
            nbytes = int(pc.sum(pc.binary_length(d)).as_py())
            dd = ST.device_dictionary(d, dev)
            target = ST.parse_target(tp)
            t_parse = timeit(lambda: K.string_parse(dd.offsets, dd.data, dd.valid, target))
            t0 = time.perf_counter()
            pc.cast(d, tp, safe=False)
            t_host = (time.perf_counter() - t0) * 1e3
            codes = torch.randint(0, m, (n,), dtype=torch.int32, device=dev)
            agg = ff.max if kind == "timestamp" else ff.sum  # SUM(CAST(s AS double)); MAX of the timestamps
            sel = SelectColumns(agg(col("s").cast(tp)).alias("x"))

            def select(dic):
                t = B200Table(Schema("s:str"), [codes], [None], {"s": dic})
                return e.select(B200DataFrame(t), sel).as_arrow()

            fresh = [pc.cast(pc.cast(d, pa.large_string()), pa.string()) for _ in range(4)]  # new dictionary objects
            select(fresh[0])
            torch.cuda.synchronize()
            first = []
            for f in fresh[1:]:
                t0 = time.perf_counter()
                select(f)
                torch.cuda.synchronize()
                first.append((time.perf_counter() - t0) * 1e3)
            t_cached = timeit(lambda: select(fresh[-1]))
            runs.append({"kind": kind, "entries": m, "entry_bytes": nbytes, "parse_ms": round(t_parse, 4),
                         "entry_GBps": round(nbytes / t_parse / 1e6, 2), "pyarrow_cast_1core_ms": round(t_host, 3),
                         "select_sum_cast_first_ms": round(sorted(first)[1], 3),
                         "select_sum_cast_cached_ms": round(t_cached, 3)})
            print(json.dumps(runs[-1]), file=sys.stderr)
            del codes, fresh
    out["dictionaries"] = runs
    # alter_columns: a 10 M-row frame of a 10 M-entry double dictionary and a long column
    m = 10_000_000
    d, _ = dictionary("double", m, 7)
    codes = torch.randint(0, m, (m,), dtype=torch.int32, device=dev)
    other = torch.arange(m, dtype=torch.int64, device=dev)
    t = B200Table(Schema("s:str,v:long"), [codes, other], [None, None], {"s": d})
    df = B200DataFrame(t)
    df.alter_columns("v:int")  # warm the other kernels; the dictionary is not parsed yet
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    df.alter_columns("s:double")
    torch.cuda.synchronize()
    t_first = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    df.alter_columns("s:double")
    torch.cuda.synchronize()
    t_dev = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    e.to_df(DataFrame.alter_columns(df, "s:double").as_arrow())
    torch.cuda.synchronize()
    t_host = (time.perf_counter() - t0) * 1e3
    out["alter_columns_10M_rows"] = {"device_first_ms": round(t_first, 2), "device_cached_ms": round(t_dev, 2),
                                     "host_round_trip_ms": round(t_host, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
