"""K10 quantiles on 100 M rows of f64 values (1 % NULL) with int64 keys, in three shapes: 10 M groups (about 10 rows
each, all on the short path), 65 536 groups (about 1 500 rows each, short path) and 256 groups (about 390 000
rows each, all on the long path).

Per shape, CUDA events, median of `--reps`:
  * ``fb_segmented_quantile`` for MEDIAN over the key-sorted column, and its algorithmic bytes (8 B value + 1 B
    validity per row, the offsets, the count and result per group) over that time;
  * the same medians through the existing radix passes: ``sort.argsort_rows`` by (key, v), then the pick (a
    gather at each group's middle rows);
  * the whole ``fa.aggregate`` with MEDIAN on the unsorted table, split into the key sort (``argsort_rows`` by
    key, the gather of the value column, ``logical_offsets``) and the quantile step, next to SUM through the hash
    group-by (K6).
The card's name and power limit are read in the same run.

    python tools/quantile_bench.py [--rows N] [--reps R] [--out FILE]
"""
import argparse
import json
import os
import sys
from collections import OrderedDict

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from fugue_b200 import kernels as K  # noqa: E402
from relational_bench import _card, timeit  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from fugue_b200 import api as fa
    from fugue_b200 import sort as S
    from fugue_b200.column import col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.table import B200Table

    dev = torch.device("cuda", 0)
    n = a.rows
    e = fa.make_execution_engine("b200")
    res = {"rows": n, "values": "f64, 1% NULL", "keys": "int64", "card": _card(dev), "shapes": {}}
    for groups in (n // 10, 1 << 16, 256):
        g = torch.Generator(device=dev).manual_seed(groups)
        key = torch.randint(0, groups, (n,), dtype=torch.int64, device=dev, generator=g)
        v = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
        valid = (torch.rand(n, device=dev, generator=g) >= 0.01).to(torch.uint8)
        t = B200Table("k:long,v:double", [key, v], [None, valid])
        r = {"groups": groups}
        # ---- the kernel on the key-sorted column
        skey, order = torch.sort(key, stable=True)
        sv, svalid = v[order].contiguous(), valid[order].contiguous()
        off = torch.zeros(groups + 1, dtype=torch.int64, device=dev)
        off[1:] = torch.cumsum(torch.bincount(skey, minlength=groups), 0)
        nseg = int((off[1:] > off[:-1]).sum())
        del skey, order
        med = [(0.5, K.QUANTILE_CONT)]
        ms = timeit(lambda: K.segmented_quantile(off, sv, svalid, K.RANGE_KEY_F64, med), reps=a.reps)
        nbytes = 9 * n + 8 * (groups + 1) + 16 * groups
        r["nonempty_groups"] = nseg
        r["kernel_ms"] = ms
        r["kernel_bytes"] = nbytes
        r["kernel_GB_per_s"] = nbytes / ms / 1e6
        # ---- the same medians through the radix passes: argsort by (key, v), then the pick
        lengths = off[1:] - off[:-1]

        def radix_median():
            idx = S.argsort_rows(t, OrderedDict(k=True, v=True))
            vs = v[idx]
            ok = valid[idx].to(torch.int64)
            cnt = torch.zeros(groups, dtype=torch.int64, device=dev)  # non-NULL values per group: NULLs sort last
            cnt.index_add_(0, key[idx], ok)
            h = 0.5 * (cnt - 1).clamp(min=0).to(torch.float64)
            lo = torch.floor(h)
            frac = h - lo
            a0 = vs[(off[:-1] + lo.to(torch.int64)).clamp(max=n - 1)]
            a1 = vs[(off[:-1] + lo.to(torch.int64) + (frac > 0).to(torch.int64)).clamp(max=n - 1)]
            return torch.where(frac == 0, a0, a0 + (a1 - a0) * frac)

        r["radix_argsort_and_pick_ms"] = timeit(radix_median, reps=a.reps)
        del lengths, sv, svalid
        torch.cuda.empty_cache()
        # ---- fa.aggregate: MEDIAN (key sort + quantile step) next to SUM through K6
        df = B200DataFrame(t)

        def key_sort():
            idx = S.argsort_rows(t, OrderedDict(k=True))
            st = S.take_rows(t, idx)
            return S.logical_offsets(st, ["k"])

        r["aggregate_median_ms"] = timeit(lambda: fa.aggregate(df, "k", m=f.median(col("v")), engine=e), reps=a.reps)
        r["aggregate_median_key_sort_ms"] = timeit(key_sort, reps=a.reps)
        r["aggregate_median_quantile_step_ms"] = r["kernel_ms"]
        r["aggregate_sum_k6_ms"] = timeit(lambda: fa.aggregate(df, "k", s=f.sum(col("v")), engine=e), reps=a.reps)
        res["shapes"][str(groups)] = r
        print(json.dumps({str(groups): r}), flush=True)
        del t, df, key, v, valid, off
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
