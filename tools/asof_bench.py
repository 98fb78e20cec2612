"""As-of join on one H100: where the time of ``fa.asof_join`` goes (DESIGN §7q, §10).

Data: left ``--left`` rows (int64 key ``k``, timestamp[us] ``t``, float64 ``v``), right ``--right`` rows (``k``,
``t``, int64 ``rid`` = its row number), with 65 536 and with 1 024 keys; direction backward, left outer.

For each key count: the whole call (CUDA events, median of ``--runs`` after one warm-up); then, in separate runs
with a device synchronise around every step, its split into right sort (``argsort_rows``), build (``JoinTable``
over the run heads), probe (``probe_counts``), search (``fb_asof_search``) and gather (the output's
``fb_gather_rows``), the rest being key surrogates, order codes and the gathers of the right keys; and, checked
equal on every left row, (a) the workaround built from existing engine calls - union of both sides with a tag, a
running LAST of ``rid`` per key ordered by (t, tag), then the left rows - and (b) ``pandas.merge_asof`` on one host core, its sorts included, on the first
``--pandas-rows`` left rows against the whole right side.  The card's name and power limit are read in the same run.

    python tools/asof_bench.py [--left N] [--right M] [--runs R] [--out result.json]
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
import pandas as pd  # noqa: E402
import torch  # noqa: E402

from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import join as J  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.column import SelectColumns, col, functions as f, lit  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.schema import Schema  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402

PHASES = {"right sort": (J, "argsort_rows"), "build": (K, "JoinTable"), "probe": (K.JoinTable, "probe_counts"),
          "search": (K, "asof_search"), "gather": (J, "_asof_assemble")}


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
    """Median milliseconds per phase, every phase function wrapped in device synchronises."""
    acc: Dict[str, List[float]] = defaultdict(list)
    saved = {name: getattr(mod, attr) for name, (mod, attr) in PHASES.items()}
    cur: Dict[str, float] = defaultdict(float)

    def wrap(name: str, inner: Callable) -> Callable:
        def run(*a: Any, **kw: Any) -> Any:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                return inner(*a, **kw)
            finally:
                torch.cuda.synchronize()
                cur[name] += (time.perf_counter() - t0) * 1e3
        return run

    try:
        for name, (mod, attr) in PHASES.items():
            setattr(mod, attr, wrap(name, saved[name]))
        fn()
        for _ in range(runs):
            cur.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            total = (time.perf_counter() - t0) * 1e3
            for name in PHASES:
                acc[name].append(cur[name])
            acc["other (key surrogates, order codes, right key gathers)"].append(total - sum(cur.values()))
    finally:
        for name, (mod, attr) in PHASES.items():
            setattr(mod, attr, saved[name])
    return {name: round(float(np.median(v)), 2) for name, v in acc.items()}


def workaround(eng: Any, left: B200DataFrame, right: B200DataFrame) -> B200DataFrame:
    """(a): union with a tag (right rows 0, so that they precede left rows of equal t), a running LAST of ``rid``
    per key ordered by (t, tag), then the left rows - which the windowed select keeps in input order."""
    n1, n2 = left.native.num_rows, right.native.num_rows
    dev = left.native.device
    lt, rt = left.native, right.native
    sch = Schema("k:long,t:datetime,tag:long,rid:long")
    u1 = B200Table(sch, [lt.column("k"), lt.column("t"), torch.ones(n1, dtype=torch.int64, device=dev),
                         torch.zeros(n1, dtype=torch.int64, device=dev)],
                   [None, None, None, torch.zeros(n1, dtype=torch.uint8, device=dev)])
    u2 = B200Table(sch, [rt.column("k"), rt.column("t"), torch.zeros(n2, dtype=torch.int64, device=dev),
                         rt.column("rid")])
    both = eng.union(B200DataFrame(u1), B200DataFrame(u2), distinct=False)
    last = f.last(col("rid")).over(rows=(None, 0), partition_by=["k"], order_by=["t", "tag"]).alias("rid")
    res = eng.select(both, SelectColumns(col("k"), col("t"), col("tag"), last))
    return eng.filter(res, col("tag") == lit(1))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--left", type=int, default=100_000_000)
    ap.add_argument("--right", type=int, default=10_000_000)
    ap.add_argument("--keys", default="65536,1024")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--pandas-rows", type=int, default=2_000_000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    n1, n2 = args.left, args.right
    eng = fa.make_execution_engine("b200")
    result: Dict[str, Any] = {"card": card(), "left": n1, "right": n2, "runs": args.runs, "cases": {}}
    for nk in [int(x) for x in args.keys.split(",")]:
        g = torch.Generator(device=dev)
        g.manual_seed(nk)
        lk = torch.randint(0, nk, (n1,), device=dev, generator=g)
        lt = torch.randint(0, 1 << 40, (n1,), device=dev, generator=g)
        lv = torch.randn(n1, device=dev, dtype=torch.float64, generator=g)
        rk = torch.randint(0, nk, (n2,), device=dev, generator=g)
        rt = torch.randint(0, 1 << 40, (n2,), device=dev, generator=g)
        left = B200DataFrame(B200Table(Schema("k:long,t:datetime,v:double"), [lk, lt, lv]))
        right = B200DataFrame(B200Table(Schema("k:long,t:datetime,rid:long"),
                                        [rk, rt, torch.arange(n2, dtype=torch.int64, device=dev)]))

        def call() -> Any:
            return eng.asof_join(left, right, on=["k"], asof="t", how="left_outer")

        case: Dict[str, Any] = {"keys": nk}
        case["asof_join_ms"] = round(timed(call, args.runs), 2)
        case["phases_ms"] = split(call, args.runs)
        out = call().native
        got = torch.where(out.valid[3].bool(), out.columns[3], torch.full_like(out.columns[3], -1))
        case["matched"] = int((got >= 0).sum())
        case["workaround_ms"] = round(timed(lambda: workaround(eng, left, right), max(1, args.runs // 2)), 2)
        w = workaround(eng, left, right).native
        wr = torch.where(w.valid[3].bool(), w.columns[3], torch.full_like(w.columns[3], -1)) \
            if w.valid[3] is not None else w.columns[3]
        case["workaround_equal"] = bool(w.num_rows == n1 and torch.equal(wr, got))
        del w, wr
        m = min(args.pandas_rows, n1)
        ldf = pd.DataFrame({"k": lk[:m].cpu().numpy(), "t": lt[:m].cpu().numpy(), "v": lv[:m].cpu().numpy()})
        rdf = pd.DataFrame({"k": rk.cpu().numpy(), "t": rt.cpu().numpy(), "rid": np.arange(n2)})
        t0 = time.perf_counter()
        ls, rs = ldf.sort_values("t", kind="stable"), rdf.sort_values("t", kind="stable")
        p = pd.merge_asof(ls, rs, on="t", by="k")
        case["pandas_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        case["pandas_rows"] = m
        pr = np.full(m, -1, dtype=np.int64)
        pr[ls.index.to_numpy()] = p["rid"].fillna(-1).to_numpy(np.int64)
        case["pandas_equal"] = bool(np.array_equal(pr, got[:m].cpu().numpy()))
        result["cases"][str(nk)] = case
        print(json.dumps(case), flush=True)
        del left, right, out, got
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
