"""Where pass 2 of the hash partition (`fb_scatter_ws_kernel`) spends its time, by ablation, on one GPU.

    python tools/scatter_breakdown.py build [--src FILE] [--tag NAME]   # compile the ablation builds (no GPU)
    python tools/scatter_breakdown.py run [--rounds 3] [--reps 12]      # time them (one GPU)
    python tools/scatter_breakdown.py profile OUT_DIR                   # torch.profiler trace of one bench step

`build` copies `fb_partition.cu` (the tree's, or --src), patches each copy by plain text replacement and compiles it
with `fb_capi.cu` into `tools/_bin/variants/<tag>-<variant>/libfb_partition.so`.  The shipped source carries no
ablation switch.  The variants (all but `base` and `linear` give wrong output; every store stays inside the output
buffers, which `run` allocates with room past their ends for the variants that misplace rows):

    base       the source unchanged (the same compile as the shipped library)
    linear     movers store slot j of a tile to row t0 + (j mod 4096): the same instructions, a linear destination
    norecords  every tile is placed by the rank record of tile 0, which stays in L2: no record traffic from HBM
    nostores   movers keep the gathered values in a register instead of storing them: the read-side floor
    noloads    the producer arrives on each ring stage instead of filling it: the write-side floor

`run` times, in one process and alternating them in every round, the shipped pass 2 (`K.partition_apply`), every
variant built, pass 1 alone (`K.partition_plan`) and a device copy of the table's 6.4 GB.  Each figure is the median
of --reps CUDA-event timings of single calls; one JSON line per figure and round, then the card, its power limit
and SM clock.  The workload is bench.py's: 100 M rows, an int64 key of 65536 values, 3 more int64 and 4 float64
columns, num = 256.
"""
import argparse
import glob
import json
import os
import shutil
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fugue_b200", "csrc")
VARIANTS_DIR = os.path.join(ROOT, "tools", "_bin", "variants")
NVCC = "/usr/local/cuda/bin/nvcc"
NVFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
           "--expt-relaxed-constexpr", "-shared", "-I", CSRC, "-I", os.path.join(ROOT, "include")]
TILE = 4096

_SINK_DECL = ("setmaxnreg_inc<kWsMoverRegs>();", "setmaxnreg_inc<kWsMoverRegs>();\n  uint64_t sink = 0;")
_SINK_USE = ("\n}\n\n// ---------------------------------------------------------------------------\n// validity bitmap",
             "\n  if (sink == 0x5EED5EED5EED5EEDull) units.dst[u0][0] = sink;  // keeps the gathers alive\n}\n\n"
             "// ---------------------------------------------------------------------------\n// validity bitmap")
# variant -> [(text in fb_partition.cu, replacement)]; each text must occur exactly once
PATCHES = {
    "base": [],
    "linear": [("dst[k] = wdelta[info >> 16] + j;", "dst[k] = (uint32_t)t0 + (j & (T - 1));")],
    "norecords": [("tma_load_1d(meta_s + b * kMetaBytes, meta + (size_t)(", "tma_load_1d(meta_s + b * kMetaBytes, meta + 0 * (size_t)(")],
    "nostores": [_SINK_DECL, _SINK_USE,
                 ("if (k0 + k < kSlotRounds && srcd[k0 + k] != 0xFFFFu) out[dst[k0 + k]] = v[k];",
                  "if (k0 + k < kSlotRounds && srcd[k0 + k] != 0xFFFFu) sink ^= v[k] + dst[k0 + k];"),
                 ("out[wpos[b] + i] = cbuf[e];", "sink ^= cbuf[e] + wpos[b];")],
    "noloads": [("mbar_expect_tx(bar_full + 8 * s, kStageBytes);\n"
                 "          tma_load_1d(ring_s + s * kStageBytes, units.src[u] + t0, kStageBytes, bar_full + 8 * s, pol);",
                 "mbar_arrive(bar_full + 8 * s);")],
}


def build(src: str, tag: str) -> None:
    text = open(src).read()
    for name, patches in PATCHES.items():
        out = text
        for old, new in patches:
            if out.count(old) != 1:
                raise SystemExit(f"{name}: the text to patch occurs {out.count(old)} times in {src}: {old[:60]!r}")
            out = out.replace(old, new)
        d = os.path.join(VARIANTS_DIR, f"{tag}-{name}")
        os.makedirs(d, exist_ok=True)
        cu = os.path.join(d, "fb_partition.cu")
        open(cu, "w").write(out)
        cmd = [NVCC, *NVFLAGS, "-o", os.path.join(d, "libfb_partition.so"), cu, os.path.join(CSRC, "fb_capi.cu")]
        print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)


def _card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia-smi": q, "value": r.stdout.strip().splitlines()[0] if r.returncode == 0 else r.stderr.strip()}


def run(rounds: int, reps: int) -> None:
    import ctypes as C

    import torch

    sys.path.insert(0, ROOT)
    from fugue_b200 import _lib
    from fugue_b200 import kernels as K

    dev = torch.device("cuda", 0)
    n, num = 100_000_000, 256
    g = torch.Generator(device=dev).manual_seed(0)
    cols = [torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)]
    cols += [torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g) for _ in range(3)]
    cols += [torch.randn(n, dtype=torch.float64, device=dev, generator=g) for _ in range(4)]
    # Room past the end of every output for the variants that misplace rows.  A partition's cursor starts inside
    # the output and a CTA advances it by at most the rows of its own tiles: chunks of the 4 groups of 2 columns
    # are dealt to S = #SM / 4 CTAs per group, at most ceil(chunks / S) chunks each.
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ntiles = n // TILE
    per_chunk = -(-ntiles // (2 * sms))
    nchunks = -(-ntiles // per_chunk)
    slack = (-(-nchunks // (sms // 4)) * per_chunk + 1) * TILE
    bufs = [torch.empty(n + slack, dtype=c.dtype, device=dev) for c in cols]
    outs = [b[:n] for b in bufs]
    plan = K.partition_plan([cols[0]], num)
    sig = _lib.SIGNATURES["fb_partition_apply_ex"]
    keys = _lib.ptr_array([cols[0].data_ptr()])
    kw = _lib.i32_array([8])
    srcs, dsts = _lib.ptr_array([c.data_ptr() for c in cols]), _lib.ptr_array([o.data_ptr() for o in outs])
    widths = _lib.i32_array([8] * len(cols))
    stream = torch.cuda.current_stream(dev).cuda_stream

    def apply_with(lib):
        fn = lib.fb_partition_apply_ex
        fn.restype, fn.argtypes = sig

        def call():
            rc = fn(0, stream, n, 1, keys, kw, None, num, plan.scratch.data_ptr(), plan.scratch.numel(),
                    plan.offsets.data_ptr(), len(cols), srcs, widths, dsts, 0, 0)
            if rc != 0:
                raise RuntimeError(lib.fb_last_error())
        return call

    figures = {"shipped pass 2 (K.partition_apply)": lambda: K.partition_apply(plan, cols, outs)}
    for d in sorted(glob.glob(os.path.join(VARIANTS_DIR, "*", "libfb_partition.so"))):
        lib = C.CDLL(d)
        lib.fb_last_error.restype = C.c_char_p
        figures[os.path.basename(os.path.dirname(d))] = apply_with(lib)
    figures["pass 1 alone (K.partition_plan)"] = lambda: K.partition_plan([cols[0]], num, scratch=plan.scratch,
                                                                         offsets=plan.offsets)
    table = torch.cat([c.view(torch.int64) for c in cols])
    copy_dst = torch.empty_like(table)
    figures["device copy of the 6.4 GB (12.8 GB moved)"] = lambda: copy_dst.copy_(table)

    def checksum():
        return [int(o.view(torch.int64).sum().item()) for o in outs] + [int(o.view(torch.int64)[n // 3].item()) for o in outs]

    ref = None
    e = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    print(json.dumps({"card": _card()}), flush=True)
    for r in range(rounds):
        for name, fn in figures.items():
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            for e0, e1 in e:
                e0.record()
                fn()
                e1.record()
            torch.cuda.synchronize()
            ms = statistics.median(a.elapsed_time(b) for a, b in e)
            line = {"round": r, "figure": name, "ms": round(ms, 4)}
            if "pass 1" not in name and "copy" not in name:
                chk = checksum()
                ref = chk if ref is None else ref
                line["same_output_as_shipped"] = chk == ref
            print(json.dumps(line), flush=True)
    print(json.dumps({"card": _card()}), flush=True)


def profile(out_dir: str) -> None:
    """One bench.py-shaped step (pass 1 + pass 2 of the 8-column table) under torch.profiler: every launch."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    sys.path.insert(0, ROOT)
    from fugue_b200 import kernels as K

    dev = torch.device("cuda", 0)
    n, num = 100_000_000, 256
    g = torch.Generator(device=dev).manual_seed(0)
    cols = [torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=dev, generator=g)]
    cols += [torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=dev, generator=g) for _ in range(7)]
    outs = [torch.empty_like(c) for c in cols]
    plan = K.partition_plan([cols[0]], num)

    def step():
        K.partition_plan([cols[0]], num, scratch=plan.scratch, offsets=plan.offsets)
        K.partition_apply(plan, cols, outs)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            step()
        torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(out_dir, "scatter_step.pt.trace.json"))
    evs = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    prev_end = None
    for ev in evs[: len(evs) // 5]:  # the first of the 5 steps, launch by launch
        gap = None if prev_end is None else round((ev.time_range.start - prev_end) / 1e3, 4)
        print(json.dumps({"kernel": ev.name[:90], "ms": round((ev.time_range.end - ev.time_range.start) / 1e3, 4),
                          "gap_before_ms": gap}), flush=True)
        prev_end = ev.time_range.end
    span = (evs[-1].time_range.end - evs[0].time_range.start) / 1e3 / 5
    print(json.dumps({"step_span_ms": round(span, 4), "launches_per_step": len(evs) // 5, "card": _card()}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("--src", default=os.path.join(CSRC, "fb_partition.cu"))
    b.add_argument("--tag", default="tree")
    b.add_argument("--clean", action="store_true", help="remove every earlier variant build first")
    r = sub.add_parser("run")
    r.add_argument("--rounds", type=int, default=3)
    r.add_argument("--reps", type=int, default=12)
    p = sub.add_parser("profile")
    p.add_argument("out_dir")
    a = ap.parse_args()
    if a.cmd == "build":
        if a.clean:
            shutil.rmtree(VARIANTS_DIR, ignore_errors=True)
        build(a.src, a.tag)
    elif a.cmd == "run":
        run(a.rounds, a.reps)
    else:
        profile(a.out_dir)


if __name__ == "__main__":
    main()
