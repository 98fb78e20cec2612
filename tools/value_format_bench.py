"""Casts to strings (K14).  Prints one JSON object; the card name and its power limit are read in the same run.  Kernel
times are medians of CUDA-event timings after a warm-up call.

- ``fb_value_format`` (measure and write call, offsets scan included) over 10 M distinct values of four kinds:
  int64, random-bit float64, two-decimal prices and timestamp[us]; as output bytes per second.
- The host formatting it replaces: Python's ``str()`` of the same 10 M values on one core, plus the ``pa.array``.
- ``fa.select(col("v").cast(str))`` over ``--rows`` rows of int64 with 1 000 and 10 M distinct values, first call
  (the dictionary is built from scratch on every call).

    python tools/value_format_bench.py [--rows N]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scalar_bench import card, timeit  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    args = ap.parse_args()
    import numpy as np
    import pyarrow as pa
    import torch

    from fugue_b200 import api as fa
    from fugue_b200 import kernels as K
    from fugue_b200.column import SelectColumns, col
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.schema import Schema
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    out = card()
    out["rows"] = args.rows
    m = 10_000_000
    rng = np.random.default_rng(14)
    kinds = {
        "int64": (rng.integers(-(1 << 62), 1 << 62, m), K.FMT_I64),
        "f64_random_bits": (rng.integers(0, 1 << 63, m).view(np.float64), K.FMT_F64),
        "f64_prices": (np.round(rng.uniform(0, 10000, m), 2), K.FMT_F64),
        "timestamp_us": (rng.integers(0, 2_000_000_000_000_000, m), K.FMT_TS + K.TU_US + K.FMT_TS_FRAC),
    }
    runs = []
    for name, (host, kind) in kinds.items():
        words = torch.from_numpy(np.ascontiguousarray(host).view(np.int64)).to(dev)
        offsets, _ = K.value_format(words, None, kind)
        nbytes = int(offsets[-1].item())
        t_dev = timeit(lambda: K.value_format(words, None, kind))
        vals = host.tolist()
        if name == "timestamp_us":
            vals = pa.array(host, pa.timestamp("us")).to_pylist()
        t0 = time.perf_counter()
        pa.array([str(v) for v in vals], type=pa.string())
        t_host = (time.perf_counter() - t0) * 1e3
        runs.append({"kind": name, "values": m, "out_bytes": nbytes, "format_ms": round(t_dev, 3),
                     "out_GBps": round(nbytes / t_dev / 1e6, 2), "host_str_1core_ms": round(t_host, 1)})
        print(json.dumps(runs[-1]), file=sys.stderr)
        del words
    out["format"] = runs
    e = fa.make_execution_engine("b200")
    sel = SelectColumns(col("v").cast(str))
    selects = []
    for distinct in (1000, 10_000_000):
        v = torch.randint(0, distinct, (args.rows,), dtype=torch.int64, device=dev) * 7919 - 12345
        df = B200DataFrame(B200Table(Schema("v:long"), [v], [None]))
        e.select(df, sel)
        torch.cuda.synchronize()
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            e.select(df, sel)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        selects.append({"distinct": distinct, "select_cast_str_first_ms": round(sorted(ts)[1], 2)})
        print(json.dumps(selects[-1]), file=sys.stderr)
        del v, df
    out["select"] = selects
    print(json.dumps(out))


if __name__ == "__main__":
    main()
