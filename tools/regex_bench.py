"""Regular expressions (K15) over a 10 M-entry dictionary of 12 to 20 ASCII bytes (letters, digits, '@', '.', '-'),
and a 100 M-row filter over it.

Medians of `--reps` (CUDA events around work that ends in a synchronise):
  * the match kernel alone (``fb_regex_match``) for a date prefix ``^\\d{4}-\\d{2}``, an e-mail-like pattern and an
    8-word alternation, with GB/s of entry bytes; the transform kernel for REGEXP_EXTRACT and a global
    REGEXP_REPLACE (measure + write calls);
  * ``fa.filter(REGEXP_MATCHES(s, 'ab'))`` next to ``fa.filter(s LIKE '%ab%')`` on the same 100 M rows, cached (the
    per-entry table is kept on the dictionary) and on a new dictionary object every call;
  * pyarrow's ``match_substring_regex`` over the same dictionary on one host core (a host figure, wall clock).
The card's name and power limit are read in the same run.

    python tools/regex_bench.py [--rows N] [--entries M] [--reps R] [--out FILE]
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

PATTERNS = {"date_prefix": r"^\d{4}-\d{2}", "email": r"[\w.]+@\w+\.\w+",
            "alternation8": "alpha|bravo|charlie|delta|echo|foxtrot|golf|hotel"}
_CHARS = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789@.-", dtype=np.uint8)


def _dictionary(n: int, seed: int) -> pa.Array:
    rng = np.random.default_rng(seed)
    lens = rng.integers(12, 21, n)
    offsets = np.zeros(n + 1, dtype=np.int32)
    np.cumsum(lens, out=offsets[1:])
    data = _CHARS[rng.integers(0, len(_CHARS), int(offsets[-1]))]
    dates = rng.random(n) < 0.25  # a quarter of the entries start with a date
    for i in np.nonzero(dates)[0][:200_000]:
        data[offsets[i]:offsets[i] + 7] = np.frombuffer(b"2024-0%d" % (i % 10), dtype=np.uint8)
    return pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offsets), pa.py_buffer(data)])


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--entries", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from fugue_b200 import api as fa
    from fugue_b200 import regex as R
    from fugue_b200 import strings as ST
    from fugue_b200.column import col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    e = fa.make_execution_engine("b200")
    d = _dictionary(a.entries, 15)
    nbytes = int(d.buffers()[2].size)
    res = {"rows": a.rows, "entries": a.entries, "entry_bytes": nbytes, "card": _card(dev), "kernels": {}}
    dd = ST.device_dictionary(d, dev)
    for name, p in PATTERNS.items():
        prog = R.match_program(p, False)
        ms = timeit(lambda: K.regex_match(dd.offsets, dd.data, dd.valid, prog), reps=a.reps)
        hits = int(K.regex_match(dd.offsets, dd.data, dd.valid, prog)[0].sum().item())
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            pc.match_substring_regex(d, pattern=p)
            ts.append((time.perf_counter() - t0) * 1e3)
        res["kernels"][name] = {"pattern": p, "match_ms": ms, "match_GBps": nbytes / ms / 1e6, "hits": hits,
                                "host_pyarrow_ms": sorted(ts)[len(ts) // 2]}
        print(json.dumps({name: res["kernels"][name]}), flush=True)
    for name, step in (("extract_email_domain", ("REGEXP_EXTRACT", r"@(\w+)", 1)),
                       ("replace_all_digits", ("REGEXP_REPLACE", r"\d+", "#", True))):
        ms = timeit(lambda: ST.apply_steps(dd.offsets, dd.data, dd.valid, [step]), reps=a.reps)
        res["kernels"][name] = {"step": list(step), "measure_scan_write_ms": ms, "GBps": nbytes / ms / 1e6}
        print(json.dumps({name: res["kernels"][name]}), flush=True)

    g = torch.Generator(device=dev).manual_seed(1)
    codes = torch.randint(0, a.entries, (a.rows,), dtype=torch.int32, device=dev, generator=g)
    df = B200DataFrame(B200Table("s:str", [codes], None, {"s": d}))
    rx, like = f.regexp_matches(col("s"), "ab"), col("s").like("%ab%")

    def fresh() -> B200DataFrame:  # the same strings as a new dictionary object: nothing cached
        return B200DataFrame(B200Table("s:str", [codes], None,
                                       {"s": pa.Array.from_buffers(d.type, len(d), d.buffers())}))

    fl = {}
    fl["filter_regex_ms"] = timeit(lambda: fa.filter(df, rx, engine=e), reps=a.reps)
    fl["filter_like_ms"] = timeit(lambda: fa.filter(df, like, engine=e), reps=a.reps)
    frames = [fresh() for _ in range(a.reps + 1)]
    fl["filter_regex_new_dictionary_ms"] = timeit(lambda: fa.filter(frames.pop(), rx, engine=e), reps=a.reps)
    frames = [fresh() for _ in range(a.reps + 1)]
    fl["filter_like_new_dictionary_ms"] = timeit(lambda: fa.filter(frames.pop(), like, engine=e), reps=a.reps)
    n_rx = int(fa.filter(df, rx, engine=e, as_fugue=True).native.num_rows)
    n_like = int(fa.filter(df, like, engine=e, as_fugue=True).native.num_rows)
    assert n_rx == n_like, (n_rx, n_like)
    fl["rows_kept"] = n_rx
    res["filter"] = fl
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
