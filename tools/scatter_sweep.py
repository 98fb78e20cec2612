"""Scatter-kernel tuning sweep (one GPU), 100 M rows x 8 columns: columns per group of the one-launch scatter
(all groups side by side in one launch), pass 1 (rank + scans), and a device-to-device copy of the same
6.4 GB as the ceiling of what the memory system moves here (read + write)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fugue_b200 import kernels as K

def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
    reps = 10
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    cols = [torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)]
    cols += [torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g) for _ in range(3)]
    cols += [torch.randn(n, dtype=torch.float64, device=dev, generator=g) for _ in range(4)]
    outs = [torch.empty_like(c) for c in cols]
    plan = K.partition_plan([cols[0]], 256)
    ref = None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for cpg in (2, 1, 4):
        for _ in range(2):
            K.partition_apply(plan, cols, outs, cols_per_launch=cpg)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            K.partition_apply(plan, cols, outs, cols_per_launch=cpg)
        e1.record(); torch.cuda.synchronize()
        chk = [int(o.view(torch.int64).sum().item()) for o in outs] + [int(outs[1][12345].item()), int(outs[5].view(torch.int64)[n - 7].item())]
        if ref is None:
            ref = chk
        print(json.dumps({"cols_per_group": cpg, "groups": -(-len(cols) // cpg), "launches": 1,
                          "ms": round(e0.elapsed_time(e1) / reps, 3), "same_output": chk == ref}), flush=True)
    for _ in range(2):
        K.partition_plan([cols[0]], 256, scratch=plan.scratch, offsets=plan.offsets)
    e0.record()
    for _ in range(reps):
        K.partition_plan([cols[0]], 256, scratch=plan.scratch, offsets=plan.offsets)
    e1.record(); torch.cuda.synchronize()
    print(json.dumps({"pass1_ms": round(e0.elapsed_time(e1) / reps, 3)}), flush=True)
    del outs, plan
    src = torch.cat([c.view(torch.int64) for c in cols])  # the table's 6.4 GB: 12.8 GB moved, as in the scatter
    dst = torch.empty_like(src)
    for _ in range(2):
        dst.copy_(src)
    e0.record()
    for _ in range(reps):
        dst.copy_(src)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print(json.dumps({"d2d_copy_GB_moved": 2 * src.numel() * 8 / 1e9, "ms": round(ms, 3),
                      "GBps_read_plus_write": round(2 * src.numel() * 8 / ms / 1e6, 1)}))

if __name__ == "__main__":
    main()
