"""Pass 1 of the hash partition (rank records + per-chunk histogram + scans) on one GPU, 100 M rows, against the
bytes it must move: a read of the key column alone (`torch.sum`) and a write of as many bytes as the rank records
(`fill_`).  Also the kBits = 4 path (num = 16), the generic key shape (two columns, one with NULLs) and the device
sort (`sort.argsort_rows` by one int64 key: one pass-1 launch per radix digit).  CUDA events, 3 warm-up calls and
20 timed calls per figure; one JSON line per figure."""
import json, os, sys
from collections import OrderedDict
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fugue_b200 import kernels as K
from fugue_b200 import sort
from fugue_b200.table import B200Table

TILE, RECORD_BYTES = 4096, 12800
REPS, WARMUP = 20, 3


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    key = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g)
    rec_bytes = (n // TILE) * RECORD_BYTES

    def out(name, ms, **kw):
        print(json.dumps({"figure": name, "ms": round(ms, 4), **kw}), flush=True)

    for num in (256, 16):
        plan = K.partition_plan([key], num)
        ms = timed(lambda: K.partition_plan([key], num, scratch=plan.scratch, offsets=plan.offsets))
        out(f"partition_plan num={num}", ms, GB=round((8 * n + rec_bytes) / 1e9, 3),
            GBps=round((8 * n + rec_bytes) / ms / 1e6, 1))
        del plan
    ms_read = timed(lambda: torch.sum(key))
    out("read floor: torch.sum(key)", ms_read, GB=round(8 * n / 1e9, 3), GBps=round(8 * n / ms_read / 1e6, 1))
    buf = torch.empty(rec_bytes, dtype=torch.uint8, device=dev)
    ms_write = timed(lambda: buf.fill_(7))
    out("write floor: fill_ of the record bytes", ms_write, GB=round(rec_bytes / 1e9, 3),
        GBps=round(rec_bytes / ms_write / 1e6, 1))
    out("sum of the two floors", ms_read + ms_write)
    del buf

    k2 = torch.randint(-1000, 1000, (n,), dtype=torch.int32, device=dev, generator=g)
    v2 = (torch.rand(n, device=dev, generator=g) > 0.1).to(torch.uint8)
    plan = K.partition_plan([key, k2], 256, [None, v2])
    ms = timed(lambda: K.partition_plan([key, k2], 256, [None, v2], scratch=plan.scratch, offsets=plan.offsets))
    out("partition_plan num=256, int64 + int32 key with NULLs", ms)
    del plan, k2, v2

    t = B200Table("key:long", [key])
    idx = sort.argsort_rows(t, OrderedDict(key=True))
    chk = int(idx[:1000].sum().item()) ^ int(idx[-1000:].sum().item())
    ms = timed(lambda: sort.argsort_rows(t, OrderedDict(key=True)))
    out("sort.argsort_rows by one int64 key", ms, check=chk)


if __name__ == "__main__":
    main()
