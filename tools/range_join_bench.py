"""Range join on one H100: where the time of ``range_join`` goes (DESIGN §7r, §10).

Data: left ``--left`` rows (int64 key ``k``, timestamp[us] ``t``, float64 ``v``), right ``--right`` intervals (``k``,
timestamp[us] ``s`` and ``e``, int64 ``rid`` = its row number) over ``--keys`` keys, inner join on ``k`` with
``s <= t < e`` (``closed="left"``), in three cases:

* (a) sessions: each key's intervals tile the time line without overlap, so a row meets about one;
* (b) overlaps: each key's intervals are 8 / (intervals a key) of the time line long, from uniform starts, so a
  row meets about six (fewer near the line's start);
* (c) nesting: each key's first interval spans the whole time line, the others are the sessions of (a) - the
  case where a walk back over a prefix maximum reads the whole run for every row.  It runs at ``--keys`` and,
  so that the runs are long, at ``--nest-keys`` keys.

For each case: the whole call (CUDA events, median of ``--runs`` after one warm-up); then, in separate runs with a
device synchronise around every step, its split into right sort (``argsort_rows``), tree (``window_tree``), count
(``fb_range_join_count``), scan (``fb_exclusive_scan_i64``), emit (``fb_range_join_emit``) and gather (the output's
``fb_gather_rows``), the rest being key surrogates, order codes and the run lookup; and the workaround -
``join`` on the key, then ``filter`` - on the largest left prefix whose key-join pairs fit ``--pair-budget``,
checked pair for pair against the range join of the same prefix.  The card's name and power limit are read in the
same run.

    python tools/range_join_bench.py [--left N] [--right M] [--keys K] [--runs R] [--case C] [--out result.json]
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
from fugue_b200 import join as J  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.column import col  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.schema import Schema  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402

PHASES = {"sort": (J, "argsort_rows"), "tree": (K, "window_tree"), "count": (K, "range_join_count"),
          "scan": (K, "exclusive_scan"), "emit": (K, "range_join_emit"), "gather": (J, "_assemble")}
SPAN = 1 << 40  # microseconds of the time line


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
            acc["other (key surrogates, order codes, run lookup)"].append(total - sum(cur.values()))
    finally:
        for name, (mod, attr) in PHASES.items():
            setattr(mod, attr, saved[name])
    return {name: round(float(np.median(v)), 2) for name, v in acc.items()}


def intervals(case: str, n2: int, nk: int, dev: torch.device, g: torch.Generator):
    """(k, s, e) of ``n2`` intervals over ``nk`` keys, about n2 / nk a key."""
    k = torch.arange(n2, dtype=torch.int64, device=dev) % nk
    cuts = torch.randint(0, SPAN, (n2,), device=dev, generator=g)
    order = torch.argsort(k * SPAN + cuts)  # per key, its cut points ascending
    k, cuts = k[order], cuts[order]
    if case == "overlaps":  # about 8 intervals over any point of a key's time line
        per_key = n2 / nk
        length = int(SPAN * 8 / per_key)
        return k, cuts, cuts + length
    first = torch.ones(n2, dtype=torch.bool, device=dev)
    first[1:] = k[1:] != k[:-1]
    nxt = torch.empty_like(cuts)
    nxt[:-1] = cuts[1:]
    last = torch.ones(n2, dtype=torch.bool, device=dev)
    last[:-1] = first[1:]
    s = torch.where(first, torch.zeros_like(cuts), cuts)  # sessions tile [0, SPAN) per key
    e = torch.where(last, torch.full_like(cuts, SPAN), nxt)
    if case == "nesting":  # the first interval of every key spans the whole line
        e = torch.where(first, torch.full_like(cuts, SPAN), e)
    return k, s, e


def pair_key(out: B200Table, n2: int) -> torch.Tensor:
    """(left row, rid) of every output row as one sortable int64."""
    return out.column("i") * n2 + out.column("rid")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--left", type=int, default=100_000_000)
    ap.add_argument("--right", type=int, default=1_000_000)
    ap.add_argument("--keys", type=int, default=65_536)
    ap.add_argument("--nest-keys", type=int, default=16)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--pair-budget", type=float, default=3e8, help="key-join pairs the workaround may build")
    ap.add_argument("--workaround-max-run", type=int, default=1024,
                    help="skip the workaround above this many intervals a key: the hash join's build walks every "
                         "earlier duplicate of a key")
    ap.add_argument("--case", default="", help="run one case only: sessions, overlaps, nesting or nesting/<keys>")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    n1, n2 = args.left, args.right
    eng = fa.make_execution_engine("b200")
    result: Dict[str, Any] = {"card": card(), "left": n1, "right": n2, "runs": args.runs, "cases": {}}
    cases = [("sessions", args.keys), ("overlaps", args.keys), ("nesting", args.keys), ("nesting", args.nest_keys)]
    if args.case:
        cases = [c for c in cases if args.case in (c[0], f"{c[0]}/{c[1]}")][:1]
    for name, nk in cases:
        g = torch.Generator(device=dev)
        g.manual_seed(nk + len(name))
        lk = torch.randint(0, nk, (n1,), device=dev, generator=g)
        lt = torch.randint(0, SPAN, (n1,), device=dev, generator=g)
        lv = torch.randn(n1, device=dev, dtype=torch.float64, generator=g)
        rk, rs, re_ = intervals(name, n2, nk, dev, g)
        rid = torch.arange(n2, dtype=torch.int64, device=dev)
        left = B200DataFrame(B200Table(Schema("k:long,t:datetime,v:double"), [lk, lt, lv]))
        right = B200DataFrame(B200Table(Schema("k:long,s:datetime,e:datetime,rid:long"), [rk, rs, re_, rid]))

        def call() -> Any:
            return eng.range_join(left, right, on=["k"], at="t", start="s", end="e", how="inner", closed="left")

        case: Dict[str, Any] = {"case": name, "keys": nk}
        case["range_join_ms"] = round(timed(call, args.runs), 2)
        case["output_rows"] = call().native.num_rows
        case["ns_per_output_row"] = round(case["range_join_ms"] * 1e6 / max(case["output_rows"], 1), 3)
        case["phases_ms"] = split(call, args.runs)
        result["cases"][f"{name}/{nk}"] = case
        if n2 / nk <= args.workaround_max_run:
            # the workaround on the largest left prefix whose key-join pairs fit the budget, checked pair for pair
            m = int(min(n1, args.pair_budget / (n2 / nk)))
            i = torch.arange(m, dtype=torch.int64, device=dev)
            lm = B200DataFrame(B200Table(Schema("k:long,t:datetime,v:double,i:long"), [lk[:m], lt[:m], lv[:m], i]))
            rng_call = lambda: eng.range_join(lm, right, on=["k"], at="t", start="s", end="e",  # noqa: E731
                                              closed="left")
            work = lambda: eng.filter(eng.join(lm, right, "inner", ["k"]),  # noqa: E731
                                      (col("s") <= col("t")) & (col("t") < col("e")))
            case["prefix_rows"] = m
            case["prefix_range_join_ms"] = round(timed(rng_call, args.runs), 2)
            case["join_filter_ms"] = round(timed(work, max(1, args.runs // 2)), 2)
            a = pair_key(rng_call().native, n2)
            b = torch.sort(pair_key(work().native, n2)).values
            case["join_filter_equal"] = bool(a.shape == b.shape and torch.equal(torch.sort(a).values, b))
            # rid ascends with s within a key, so the promised order is ascending (left row, rid)
            case["range_join_pairs_in_order"] = bool(a.shape[0] < 2 or bool((a[1:] >= a[:-1]).all()))
            del a, b, lm, i
        print(json.dumps(case), flush=True)
        del left, right, lk, lt, lv, rk, rs, re_, rid
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
