"""LIKE and LENGTH (K11 + FB_X_LOOKUP in K8) on 100 M rows of a dictionary-encoded string column, with
dictionaries of 1 000 and 10 M entries of 12 to 20 ASCII bytes (16 on average).

Per dictionary, medians of `--reps` (CUDA events around work that ends in a synchronise):
  * the per-entry kernels alone: ``fb_string_like`` for '%ab%' and ``fb_string_length``;
  * the dictionary upload: ``fa.filter`` on a table whose dictionary is a new object every call (so every call
    uploads it), next to the same call with the cached copy, and the upload alone;
  * ``fa.filter(col("s").like("%ab%"))`` next to ``fa.filter(col("s") == "x")`` on the same table;
  * a ``LENGTH`` select;
  * pyarrow's ``pc.match_like`` over the same dictionary on one host core (a host figure, wall clock).
The card's name and power limit are read in the same run.

    python tools/string_bench.py [--rows N] [--reps R] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import pyarrow.compute as pc  # noqa: E402
import torch  # noqa: E402

from fugue_b200 import kernels as K  # noqa: E402
from relational_bench import _card, timeit  # noqa: E402


def _dictionary(n: int, seed: int) -> pa.Array:
    """n strings of 12..20 lowercase ASCII letters, built straight into Arrow buffers."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(12, 21, n)
    offsets = np.zeros(n + 1, dtype=np.int32)
    np.cumsum(lens, out=offsets[1:])
    data = rng.integers(ord("a"), ord("z") + 1, int(offsets[-1]), dtype=np.uint8)
    return pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offsets), pa.py_buffer(data)])


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from fugue_b200 import api as fa
    from fugue_b200 import strings as ST
    from fugue_b200.column import SelectColumns, col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    n = a.rows
    e = fa.make_execution_engine("b200")
    res = {"rows": n, "strings": "12-20 ASCII bytes", "card": _card(dev), "dictionaries": {}}
    for ndict in (1000, 10_000_000):
        d = _dictionary(ndict, ndict)
        g = torch.Generator(device=dev).manual_seed(ndict)
        codes = torch.randint(0, ndict, (n,), dtype=torch.int32, device=dev, generator=g)
        t = B200Table("s:str", [codes], None, {"s": d})
        df = B200DataFrame(t)
        like = col("s").like("%ab%")
        r = {"entries": ndict, "dictionary_bytes": int(d.buffers()[2].size) + 4 * (ndict + 1)}
        dd = ST.device_dictionary(d, dev)
        toks = ST.like_tokens("%ab%", None)
        r["kernel_like_ms"] = timeit(lambda: K.string_like(dd.offsets, dd.data, dd.valid, toks), reps=a.reps)
        r["kernel_length_ms"] = timeit(lambda: K.string_length(dd.offsets, dd.data, dd.valid), reps=a.reps)

        def fresh() -> B200DataFrame:  # the same strings as a new dictionary object: not in the cache
            return B200DataFrame(B200Table("s:str", [codes], None,
                                           {"s": pa.Array.from_buffers(d.type, len(d), d.buffers())}))

        r["upload_ms"] = timeit(lambda: ST._upload(d, dev), reps=a.reps)
        frames = [fresh() for _ in range(a.reps + 1)]
        r["filter_like_first_call_ms"] = timeit(lambda: fa.filter(frames.pop(), like, engine=e), reps=a.reps)
        r["filter_like_ms"] = timeit(lambda: fa.filter(df, like, engine=e), reps=a.reps)
        r["filter_like_rows"] = int(fa.filter(df, like, engine=e, as_fugue=True).native.num_rows)
        lit = d[ndict // 2].as_py()
        r["filter_eq_ms"] = timeit(lambda: fa.filter(df, col("s") == lit, engine=e), reps=a.reps)
        sel = SelectColumns(f.length(col("s")).alias("n"))
        r["select_length_ms"] = timeit(lambda: e.select(df, sel), reps=a.reps)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            pc.match_like(d, "%ab%")
            ts.append((time.perf_counter() - t0) * 1e3)
        r["host_pyarrow_match_like_dictionary_ms"] = sorted(ts)[len(ts) // 2]
        res["dictionaries"][str(ndict)] = r
        print(json.dumps({str(ndict): r}), flush=True)
        del t, df, codes, dd, frames
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
