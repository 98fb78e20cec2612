"""Secondary measurements: BASELINE configs 4 (GROUP BY) and 5 (JOIN) at single-GPU scale."""
import os, sys, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fugue_b200 import kernels as K

def timeit(fn, reps=3):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]

def measure(device_index: int = 0):
    dev = torch.device("cuda", device_index)
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    n, nk = 125_000_000, 10_000_000      # config 4 per-GPU share of 1B rows / 8 GPUs
    keys = torch.randint(0, nk, (n,), dtype=torch.int64, device=dev, generator=g) * 0x9E3779B97F4A7C15 % (1 << 62)
    v = torch.randn(n, dtype=torch.float64, device=dev, generator=g).view(torch.int64)
    ms = timeit(lambda: K.groupby_u64(keys, None, [v, None], [None, None], [K.AGG_SUM_F64, K.AGG_COUNT]))
    out["groupby_sum_count"] = {"rows": n, "distinct_keys": nk, "ms": ms, "rows_per_s": n / ms * 1e3,
                                "alg_GBps": 16 * n / ms / 1e6}
    del keys, v
    n = 62_500_000                        # config 5 per-GPU share: 500M x 500M / 8
    lk = torch.randint(0, n, (n,), dtype=torch.int64, device=dev, generator=g)
    rk = torch.randperm(n, dtype=torch.int64, device=dev, generator=g)
    lv = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    rv = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    def join():
        tab = K.JoinTable(rk, None)
        li, ri = tab.probe(lk, None, outer=False)
        K.gather_rows([lk, lv], [None, None], li, False)
        K.gather_rows([rv], [None], ri, False)
    ms_flat = timeit(join)
    from fugue_b200 import api as fa
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.table import B200Table
    e = fa.make_execution_engine("b200")
    L = B200DataFrame(B200Table("key:long,lv:double", [lk, lv]))
    R = B200DataFrame(B200Table("key:long,rv:double", [rk, rv]))
    res = e.join(L, R, "inner", ["key"])
    assert res.count() == n
    ms = timeit(lambda: e.join(L, R, "inner", ["key"]))
    out["inner_join_flat_table_ms"] = ms_flat
    out["inner_join"] = {"left_rows": n, "right_rows": n, "out_rows": n, "ms": ms, "out_rows_per_s": n / ms * 1e3,
                         "alg_GBps": 56 * n / ms / 1e6}
    del lk, rk, lv, rv, L, R, res
    # K8: one-pass expression evaluation (SELECT list) and a WHERE filter, 100 M rows
    from fugue_b200.column import SelectColumns, col
    n = 100_000_000
    key = torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)
    v0 = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    v1 = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    T = B200DataFrame(B200Table("key:long,v0:double,v1:double", [key, v0, v1]))
    sel = SelectColumns((col("v0") * col("v1") + col("key")).alias("x"),
                        ((col("v0") > 0) & (col("v1") < 0.5)).alias("p"),
                        (col("key") * 3 - 7).alias("k3"))
    ms = timeit(lambda: e.select(T, sel))
    out["select_3_exprs"] = {"rows": n, "ms": ms, "rows_per_s": n / ms * 1e3,
                             "alg_GBps": (24 + 8 + 1 + 8) * n / ms / 1e6}   # read 3 cols once, write f64 + bool + i64
    cond = (col("v0") > 0.5) & (col("key") < 60000)
    kept = e.filter(T, cond).count()
    ms = timeit(lambda: e.filter(T, cond))
    out["filter"] = {"rows": n, "kept": kept, "ms": ms, "rows_per_s": n / ms * 1e3,
                     "alg_GBps": (16 * n + 2 * 24 * kept) / ms / 1e6}      # predicate columns + gather of kept rows
    del key, v0, v1, T
    # skewed variant of the headline workload (SURVEY.md 8d): keys Zipf(s = 1.0) over 2^16 values
    n = 100_000_000
    w = 1.0 / torch.arange(1, (1 << 16) + 1, dtype=torch.float64, device=dev)
    cdf = torch.cumsum(w, 0) / w.sum()
    zkey = torch.searchsorted(cdf, torch.rand(n, dtype=torch.float64, device=dev, generator=g)).clamp_(max=(1 << 16) - 1)
    cols = [zkey] + [torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g) for _ in range(3)] \
        + [torch.randn(n, dtype=torch.float64, device=dev, generator=g) for _ in range(4)]
    outs = [torch.empty_like(c) for c in cols]
    scratch = torch.empty(K.partition_scratch_bytes(dev, n, 256) + 256, dtype=torch.uint8, device=dev)
    off = torch.empty(257, dtype=torch.int64, device=dev)
    ms = timeit(lambda: K.partition_columns(cols, [0], 256, out=outs, scratch=scratch, offsets=off), reps=5)
    sizes = (off[1:] - off[:-1])
    pid = K.partition_ids([outs[0]], 256).long()
    ok = bool((pid == torch.repeat_interleave(torch.arange(256, device=dev), sizes)).all()) and int(off[-1]) == n
    # K4: the fused map epilogue - hash partition + map (w = v0*2 + v1 replaces v1) in one pass, beside identity
    from fugue_b200.colmap import ColumnMap
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.column import col as _c
    g2 = torch.Generator(device=dev).manual_seed(3)
    ucols = [torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g2)] \
        + [torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g2) for _ in range(3)] \
        + [torch.randn(n, dtype=torch.float64, device=dev, generator=g2) for _ in range(4)]
    names = ["key", "i1", "i2", "i3", "v0", "v1", "v2", "v3"]
    U = B200DataFrame(B200Table("key:long,i1:long,i2:long,i3:long,v0:double,v1:double,v2:double,v3:double", ucols))
    spec = PartitionSpec(by="key", algo="hash", num=256)
    cm_id = ColumnMap(*names)
    cm = ColumnMap("key", "i1", "i2", "i3", "v0", (_c("v0") * 2 + _c("v1")).alias("w"), "v2", "v3")
    sch_map = "key:long,i1:long,i2:long,i3:long,v0:double,w:double,v2:double,v3:double"
    ms_id = timeit(lambda: fa.transform(U, cm_id, schema="*", partition=spec, engine=e), reps=5)
    ms_map = timeit(lambda: fa.transform(U, cm, schema=sch_map, partition=spec, engine=e), reps=5)
    ms_unfused = timeit(lambda: cm(e.repartition(U, spec).native), reps=3)
    out["transform_fused_map"] = {"rows": n, "map": "w = v0 * 2 + v1 (7 columns copied)", "identity_ms": ms_id,
                                  "fused_map_ms": ms_map, "partition_then_evaluator_ms": ms_unfused,
                                  "rows_per_s": n / ms_map * 1e3, "alg_GBps": (64 + 64) * n / ms_map / 1e6}
    del ucols, U
    out["transform_window"] = measure_window(dev, e, n)
    out["transform_zipf_s1"] = {"rows": n, "ms": ms, "rows_per_s": n / ms * 1e3, "largest_partition_share":
                                float(sizes.max()) / n, "every_row_in_its_partition": ok}
    return out


def _card(dev):
    """Name and power limit of the card, read in the same run as the numbers they qualify."""
    info = {"name": torch.cuda.get_device_name(dev)}
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(dev.index)
        info["power_limit_w"] = nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception as ex:  # pragma: no cover
        info["power_limit_w"] = f"unavailable: {type(ex).__name__}"
    return info


def measure_window(dev, e, n):
    """K9: window functions over the logical partitions of the headline table (100 M rows, key over 2^16 values):
    a running sum, a row number, a lag and a share of the partition total, PartitionSpec(by=key, presort=i1, num=256).
    The whole call and its steps - sort by (key, presort), hash partition, window step (logical offsets, argument
    columns, scans, gathers), evaluator - and fb_segmented_scan alone."""
    from collections import OrderedDict
    from fugue_b200 import api as fa
    from fugue_b200 import expr as X
    from fugue_b200 import sort as S
    from fugue_b200.colmap import ColumnMap, _with_windows
    from fugue_b200.column import col, functions as f
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.table import B200Table
    g = torch.Generator(device=dev).manual_seed(4)
    cols = [torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g),
            torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g),
            torch.randn(n, dtype=torch.float64, device=dev, generator=g),
            torch.randn(n, dtype=torch.float64, device=dev, generator=g)]
    T = B200DataFrame(B200Table("key:long,i1:long,v0:double,v1:double", cols))
    spec = PartitionSpec(by="key", presort="i1", num=256)
    cm = ColumnMap("key", "i1", "v0", f.sum(col("v0")).over(running=True).alias("run_v0"),
                   f.row_number().alias("rn"), f.lag(col("v1")).alias("prev_v1"),
                   (col("v0") / f.sum(col("v0")).over()).alias("share"))
    schema = "key:long,i1:long,v0:double,run_v0:double,rn:long,prev_v1:double,share:double"
    ms_call = timeit(lambda: fa.transform(T, cm, schema=schema, partition=spec, engine=e))
    order = OrderedDict([("key", True), ("i1", True)])
    srt = S.sort_table(T.native, order)
    ms_sort = timeit(lambda: S.sort_table(T.native, order))
    ms_part = timeit(lambda: e.repartition(B200DataFrame(srt), spec))
    part = e.repartition(B200DataFrame(srt), spec).native
    del srt
    sel = cm.select(part).all_cols

    def window_step():
        part.logical_offsets = S.logical_offsets(part, ["key"])
        part.logical_order = ["i1"]
        return _with_windows(part, sel)
    ms_window = timeit(window_step)
    src = window_step()
    outs = [X.rewrite(c, src.window_column) for c in sel]
    ms_eval = timeit(lambda: X.project(src, outs))
    off = part.logical_offsets
    v0 = part.column("v0")
    scans = [(K.AGG_SUM_F64, v0, None), (K.AGG_SUM_F64, v0, None)]  # the running and the partition sum
    ms_scan = timeit(lambda: K.segmented_scan(off, n, scans), reps=10)
    alg_bytes = len(scans) * n * (8 + 8 + 8)   # read the value, write the value and the count
    return {"rows": n, "partitions": int(off.shape[0]) - 1,
            "map": "SUM(v0) running, ROW_NUMBER, LAG(v1), v0 / SUM(v0) over the partition",
            "ms": ms_call, "rows_per_s": n / ms_call * 1e3, "sort_ms": ms_sort, "partition_ms": ms_part,
            "window_step_ms": ms_window, "evaluator_ms": ms_eval,
            "segmented_scan": {"ms": ms_scan, "scans": len(scans), "alg_bytes": alg_bytes,
                               "alg_GBps": alg_bytes / ms_scan / 1e6,
                               "share_of_3350_GBps": alg_bytes / ms_scan / 1e6 / 3350.0,
                               "bytes_moved": len(scans) * n * 32,
                               "note": "reduce-then-scan reads every value twice: 32 B per row and scan move"},
            "card": _card(dev)}


def _dist_time(fn, dev, reps=3):
    """CUDA-event time of a collective step: barrier + synchronize on both sides, max over ranks, median of reps."""
    import torch.distributed as dist

    fn(); torch.cuda.synchronize(dev)
    ts = []
    for _ in range(reps):
        dist.barrier(); torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(dev)
        t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ts.append(float(t.item()))
    return sorted(ts)[len(ts) // 2]


def measure_dist(engine, rank, world, dev):
    """BASELINE configs 4 and 5 on `world` GPUs (every rank calls this): per-GPU share of 1 B-row GROUP BY
    (10 M distinct keys) and of 500 M x 500 M inner join, through DistributedB200Engine.aggregate / .join."""
    import torch.distributed as dist
    from fugue_b200.column import all_cols, col, functions as ff
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.table import B200Table

    g = torch.Generator(device=dev).manual_seed(1234 + rank)
    out = {"n_gpus": world}
    n, nk = 125_000_000, 10_000_000
    keys = torch.randint(0, nk, (n,), dtype=torch.int64, device=dev, generator=g) * 0x9E3779B97F4A7C15 % (1 << 62)
    v = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    T = B200DataFrame(B200Table("key:long,v0:double", [keys, v]))
    spec = PartitionSpec(by=["key"])
    aggs = [ff.sum(col("v0")).alias("s"), ff.count(all_cols()).alias("c")]
    res = engine.aggregate(T, spec, aggs)
    cnt = torch.tensor([res.count(), int(res.native.column("c").sum().item())], dtype=torch.int64, device=dev)
    dist.all_reduce(cnt)
    ms = _dist_time(lambda: engine.aggregate(T, spec, aggs), dev)
    out["groupby_sum_count"] = {"rows": n * world, "rows_per_gpu": n, "distinct_keys": nk, "groups_out": int(cnt[0]),
                                "count_total_matches_rows": int(cnt[1]) == n * world, "ms": ms,
                                "rows_per_s": n * world / ms * 1e3, "alg_GBps_per_gpu": 16 * n / ms / 1e6,
                                "config": "BASELINE config 4 share: SELECT key, SUM(v0), COUNT(*) GROUP BY key"}
    del keys, v, T, res
    torch.cuda.empty_cache()
    n = 62_500_000
    total = n * world
    lk = torch.randint(0, total, (n,), dtype=torch.int64, device=dev, generator=g)
    # unique build side: an affine bijection of [0, total) (a coprime to total), sharded by row range
    a_mul = 2_654_435_761
    while total % 2 == 0 and a_mul % 2 == 0:
        a_mul += 1
    import math
    while math.gcd(a_mul, total) != 1:
        a_mul += 2
    idx = torch.arange(rank * n, (rank + 1) * n, dtype=torch.int64, device=dev)
    rk = (idx * a_mul + 12345) % total
    lv = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    rv = torch.randn(n, dtype=torch.float64, device=dev, generator=g)
    L = B200DataFrame(B200Table("key:long,lv:double", [lk, lv]))
    R = B200DataFrame(B200Table("key:long,rv:double", [rk, rv]))
    res = engine.join(L, R, "inner", ["key"])
    cnt = torch.tensor([res.count()], dtype=torch.int64, device=dev)
    dist.all_reduce(cnt)
    del res
    ms = _dist_time(lambda: engine.join(L, R, "inner", ["key"]), dev)
    out["inner_join"] = {"left_rows": total, "right_rows": total, "out_rows": int(cnt[0]), "rows_per_gpu": n,
                         "out_rows_equals_left_rows": int(cnt[0]) == total, "ms": ms,
                         "out_rows_per_s": total / ms * 1e3, "alg_GBps_per_gpu": 56 * n / ms / 1e6,
                         "config": "BASELINE config 5 share: inner join on int64 key, unique build side"}
    return out


def cpu_baselines():
    """pandas (what the reference's native engine runs: qpd -> groupby.agg; triad -> pd.merge) on bounded
    samples of configs 4 / 5, 1 core."""
    import numpy as np
    import pandas as pd

    rng = np.random.default_rng(0)
    n, nk = 20_000_000, 1_600_000   # same 12.5 rows per key as 125 M rows / 10 M keys
    kk = (rng.integers(0, nk, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) % np.uint64(1 << 62)
    df = pd.DataFrame({"key": kk.astype(np.int64), "v0": rng.standard_normal(n)})
    t0 = time.perf_counter()
    r = df.groupby("key").agg(s=("v0", "sum"), c=("v0", "size"))
    t_g = time.perf_counter() - t0
    m = 10_000_000
    left = pd.DataFrame({"key": rng.integers(0, m, m), "lv": rng.standard_normal(m)})
    right = pd.DataFrame({"key": rng.permutation(m), "rv": rng.standard_normal(m)})
    t0 = time.perf_counter()
    j = left.merge(right, on="key", how="inner")
    t_j = time.perf_counter() - t0
    return {"kind": "port", "cores": 1,
            "groupby": {"rows": n, "groups": len(r), "s": t_g, "rows_per_s": n / t_g, "sample": "20 M rows, 1.6 M keys "
                        "(the workload's 12.5 rows per key), pandas groupby.agg(sum, size)"},
            "inner_join": {"rows": m, "out_rows": len(j), "s": t_j, "out_rows_per_s": len(j) / t_j,
                           "sample": "10 M x 10 M rows, unique build side, pandas merge"}}


if __name__ == "__main__":
    print(json.dumps(measure()))
