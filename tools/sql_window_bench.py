"""Window functions in SQL on one H100: where the time of a windowed SELECT goes (DESIGN §7p, §10).

Data: 100 M rows, an int64 key ``k`` with 65 536 distinct values, an int64 ``t`` and a float64 ``v``.  Queries:

    (a) SELECT k, t, v FROM df QUALIFY ROW_NUMBER() OVER (PARTITION BY k ORDER BY t DESC) = 1
    (b) SELECT k, v / SUM(v) OVER (PARTITION BY k) AS share FROM df
    (c) SELECT k, AVG(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) AS m FROM df

For each: the whole call (CUDA events, median of ``--runs`` after one warm-up), then, in separate runs with a device
synchronise around every step, its split into sort (``argsort_rows``), gather (``take_rows``), window kernels
(``_with_windows``), scatter-back (``fb_scatter_rows``) and projection (evaluator passes, the QUALIFY filter);
the same result through ``fa.transform(ColumnMap)``; and ``fb_scatter_rows`` against an inverse permutation plus
``fb_gather_rows``, the route it replaces.  The card's name, power limit and SM clock are read in the same run.

    python tools/sql_window_bench.py [--rows N] [--runs R] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict
from typing import Any, Callable, Dict, List

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import colmap as CM  # noqa: E402
from fugue_b200 import expr as X  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200 import sort as S  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import col, functions as f  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.schema import Schema  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402

QUERIES = {
    "a_qualify_latest": ("SELECT k, t, v FROM", "QUALIFY ROW_NUMBER() OVER (PARTITION BY k ORDER BY t DESC) = 1"),
    "b_share": ("SELECT k, v / SUM(v) OVER (PARTITION BY k) AS share FROM", ""),
    "c_moving_avg": ("SELECT k, AVG(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) "
                     "AS m FROM", ""),
}
MAPS = {  # the same windows through the ColumnMap route
    "a_qualify_latest": (["k", "t", "v", f.row_number().alias("rn")], "k:long,t:long,v:double,rn:long", "t desc"),
    "b_share": (["k", (col("v") / f.sum(col("v")).over()).alias("share")], "k:long,share:double", None),
    "c_moving_avg": (["k", f.avg(col("v")).over(rows=(-6, 0)).alias("m")], "k:long,m:double", "t"),
}
PHASES = {"sort": (S, "argsort_rows"), "gather": (S, "take_rows"), "window kernels": (CM, "_with_windows"),
          "scatter-back": (CM, "_to_input_order"), "projection": (X, "project"), "qualify filter": (X, "filter_table")}


def card() -> Dict[str, str]:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def timed(fn: Callable[[], Any], runs: int) -> float:
    """Median milliseconds of ``fn`` between CUDA events, after one warm-up call."""
    fn()
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def split(fn: Callable[[], Any], runs: int) -> Dict[str, float]:
    """Median milliseconds per phase: every phase function wrapped in device synchronises (outermost call only,
    so the gathers inside the window kernels' finishers count as window kernels)."""
    acc: Dict[str, List[float]] = defaultdict(list)
    saved = {name: getattr(mod, attr) for name, (mod, attr) in PHASES.items()}
    depth = [0]

    def wrap(name: str, inner: Callable) -> Callable:
        def run(*a: Any, **kw: Any) -> Any:
            if depth[0]:
                return inner(*a, **kw)
            depth[0] += 1
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                return inner(*a, **kw)
            finally:
                torch.cuda.synchronize()
                cur[name] += (time.perf_counter() - t0) * 1e3
                depth[0] -= 1
        return run

    cur: Dict[str, float] = defaultdict(float)
    try:
        for name, (mod, attr) in PHASES.items():
            setattr(mod, attr, wrap(name, saved[name]))
        fn()
        for _ in range(runs):
            cur = defaultdict(float)
            fn()
            for name in PHASES:
                acc[name].append(cur[name])
    finally:
        for name, (mod, attr) in PHASES.items():
            setattr(mod, attr, saved[name])
    return {name: float(np.median(v)) for name, v in acc.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--keys", type=int, default=65_536)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.rows
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    k = torch.randint(0, args.keys, (n,), device=dev, generator=g)
    t = torch.randint(0, 1 << 40, (n,), device=dev, generator=g)
    v = torch.randn(n, device=dev, dtype=torch.float64, generator=g)
    df = B200DataFrame(B200Table(Schema("k:long,t:long,v:double"), [k, t, v]))
    eng = fa.make_execution_engine("b200")
    result: Dict[str, Any] = {"card": card(), "rows": n, "keys": args.keys, "runs": args.runs, "queries": {}}
    for name, (head, tail) in QUERIES.items():
        def sql() -> Any:
            return fa.raw_sql(head, df, tail, engine=eng, as_fugue=True)

        cols, schema, presort = MAPS[name]
        spec = PartitionSpec(by=["k"], presort=presort) if presort else PartitionSpec(by=["k"])

        def cmap() -> Any:
            return fa.transform(df, ColumnMap(*cols), schema=schema, partition=spec, engine=eng, as_fugue=True)

        rows_out = sql().native.num_rows
        total = timed(sql, args.runs)
        result["queries"][name] = {"sql": f"{head} df {tail}".strip(), "rows_out": rows_out, "total_ms": total,
                                   "split_ms": split(sql, args.runs), "column_map_ms": timed(cmap, args.runs)}
        torch.cuda.empty_cache()
    # scatter-back: one fb_scatter_rows launch against inverse permutation (index_put) + fb_gather_rows
    tb = B200Table(Schema("k:long,t:long"), [k, t])
    from collections import OrderedDict

    idx = S.argsort_rows(tb, OrderedDict([("k", True), ("t", False)]))
    inv_cmp: Dict[str, Any] = {}
    for ncols in (1, 2, 3):
        src = [torch.randn(n, device=dev, dtype=torch.float64, generator=g) for _ in range(ncols)]
        valid: List[Any] = [None] * ncols
        ar = torch.arange(n, device=dev, dtype=torch.int64)

        def inverse_gather() -> Any:
            inv = torch.empty_like(idx)
            inv[idx] = ar
            return K.gather_rows(src, valid, inv, want_valid=False)

        a, b = K.scatter_rows(src, valid, idx)[0], inverse_gather()[0]
        assert all(torch.equal(x, y) for x, y in zip(a, b)), "scatter and inverse + gather differ"
        inv_cmp[f"{ncols}_f64_columns"] = {"scatter_rows_ms": timed(lambda: K.scatter_rows(src, valid, idx), args.runs),
                                           "inverse_plus_gather_ms": timed(inverse_gather, args.runs)}
        del src
    result["scatter_vs_inverse_gather"] = inv_cmp
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
