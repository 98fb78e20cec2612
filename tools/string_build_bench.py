"""UPPER / LOWER (K12 + FB_X_LOOKUP in K8) on 100 M rows of a dictionary-encoded string column, with
dictionaries of 1 000 and 10 M entries of 12 to 20 ASCII bytes (16 on average), as tools/string_bench.py.

Per dictionary, medians of `--reps` (CUDA events around work that ends in a synchronise):
  * the transform alone: the measure and write calls of ``fb_string_transform`` (UPPER) and the host scan;
  * the deduplication of the transformed entries (hash, radix sort, first-equal, gather) without and with
    the copy to the host (D2H and the ``pa.Array``);
  * ``fa.select(UPPER(s))`` on a dictionary that is a new object every call (the first call), and cached;
  * ``GROUP BY LOWER(s)`` with ``COUNT(*)`` (cached);
  * pyarrow's ``pc.utf8_upper`` over the same dictionary on one host core (a host figure, wall clock).
The card's name and power limit are read in the same run.

    python tools/string_build_bench.py [--rows N] [--reps R] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import pyarrow as pa  # noqa: E402
import pyarrow.compute as pc  # noqa: E402
import torch  # noqa: E402

from relational_bench import _card, timeit  # noqa: E402
from string_bench import _dictionary  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from fugue_b200 import api as fa
    from fugue_b200 import kernels as K
    from fugue_b200 import strings as ST
    from fugue_b200.column import SelectColumns, col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.sort import _radix_sort_pairs
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    n = a.rows
    e = fa.make_execution_engine("b200")
    res = {"rows": n, "strings": "12-20 ASCII bytes", "card": _card(dev), "dictionaries": {}}
    upper = SelectColumns(f.upper(col("s")).alias("u"))
    group = SelectColumns(f.lower(col("s")).alias("l"), f.count(col("*")).alias("n"))
    for ndict in (1000, 10_000_000):
        d = _dictionary(ndict, ndict)
        g = torch.Generator(device=dev).manual_seed(ndict)
        codes = torch.randint(0, ndict, (n,), dtype=torch.int32, device=dev, generator=g)
        df = B200DataFrame(B200Table("s:str", [codes], None, {"s": d}))
        r = {"entries": ndict}
        dd = ST.device_dictionary(d, dev)
        _, steps = ST.string_chain(f.upper(col("s")), {"s"})
        r["transform_upper_ms"] = timeit(lambda: ST.apply_steps(dd.offsets, dd.data, dd.valid, steps), reps=a.reps)
        o, dt, v = ST.apply_steps(dd.offsets, dd.data, dd.valid, steps)

        def dedup_device() -> None:
            ids = torch.arange(ndict, dtype=torch.int64, device=dev)
            sh, si = _radix_sort_pairs(K.string_hash(o, dt, v), ids)  # (sorts ids in place)
            K.string_first_equal(o, dt, v, sh, si)

        r["dedup_device_ms"] = timeit(dedup_device, reps=a.reps)
        r["dedup_with_d2h_ms"] = timeit(lambda: ST.dedup(o, dt, v), reps=a.reps)

        def fresh() -> B200DataFrame:  # the same strings as a new dictionary object: nothing cached
            return B200DataFrame(B200Table("s:str", [codes], None,
                                           {"s": pa.Array.from_buffers(d.type, len(d), d.buffers())}))

        frames = [fresh() for _ in range(a.reps + 1)]
        r["select_upper_first_call_ms"] = timeit(lambda: e.select(frames.pop(), upper), reps=a.reps)
        r["select_upper_cached_ms"] = timeit(lambda: e.select(df, upper), reps=a.reps)
        r["select_length_ms"] = timeit(lambda: e.select(df, SelectColumns(f.length(col("s")).alias("n"))),
                                       reps=a.reps)
        r["group_by_lower_ms"] = timeit(lambda: e.select(df, group), reps=a.reps)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            pc.utf8_upper(d)
            ts.append((time.perf_counter() - t0) * 1e3)
        r["host_pyarrow_utf8_upper_dictionary_ms"] = sorted(ts)[len(ts) // 2]
        res["dictionaries"][str(ndict)] = r
        print(json.dumps({str(ndict): r}), flush=True)
        del df, codes, dd, frames, o, dt, v
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
