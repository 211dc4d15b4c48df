#!/usr/bin/env python
"""The closure call (mm_kernel_enqueue_closure) against the workaround it replaces, on one GPU.

    python scripts/bench_closure.py [--seconds 1.0] [--rounds 3] [--workload NAME ...] [--json FILE]

Three arms per workload, on the same device buffers:
  closure   enqueue_closure: blocked Floyd-Warshall in place (about 2 N^3 Map / Reduce operations)
  squaring  D <- D (+) D (x) D through enqueue_accumulate into a copy, ceil(log2 N) times (what the existing API offers)
  plain     one plain N^3 product of the same semiring (the yardstick for 2 N^3 operations)
Workloads: float (Add, Min) N = 8192, int32 (Add, Min) N = 8192, a batch of 1024 float (Add, Min) graphs of 256
vertices.  The data are integer weights 1 .. 999, so that every path sum is exact: the closure and squaring to a fixed
point must write identical bytes (checked once per workload).  Each arm is warmed up, then the arms are timed
alternately, `--rounds` windows each of at least `--seconds` of device work (CUDA events); the median window is
reported as milliseconds per call.  Afterwards one closure call per workload runs under torch.profiler, and the kernel
time is split by phase (pivot, panel, remainder).  The card's name, power limit and SM clock limit are read in the same
run.  Needs a CUDA device; no fallback.
"""
import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402
import gemm_hls_b200 as G  # noqa: E402
from bench_accumulate import gpu_info, window  # noqa: E402

# name: (dtype, N, batch)
WORKLOADS = {
    "float_addmin_8192": (G.FLOAT, 8192, 1),
    "int32_addmin_8192": (G.INT32, 8192, 1),
    "float_addmin_256_x1024": (G.FLOAT, 256, 1024),
}
TORCH_DTYPE = {G.FLOAT: torch.float32, G.INT32: torch.int32}
PHASES = (("pivot", "semiring_closure_pivot_kernel"), ("panel", "semiring_closure_panel_kernel"),
          ("remainder", "semiring_closure_ring_kernel"))


def bench(ctx, name, seconds, rounds):
    dt, n, batch = WORKLOADS[name]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    d0 = torch.randint(1, 1000, (batch, n, n), generator=gen, device="cuda", dtype=torch.int32).to(TORCH_DTYPE[dt])
    d, x, y, tmp = d0.clone(), d0.clone(), torch.empty_like(d0), torch.empty_like(d0)
    s = torch.cuda.current_stream().cuda_stream
    squarings = math.ceil(math.log2(n))

    def closure():
        ctx.enqueue_closure(dt, G.ADD, G.MIN, d.data_ptr(), n, batch, stream=s)

    def squaring():
        src, dst = x, y
        for _ in range(squarings):
            dst.copy_(src)
            ctx.enqueue_accumulate(dt, G.ADD, G.MIN, src.data_ptr(), src.data_ptr(), dst.data_ptr(), n, n, n, batch,
                                   stream=s)
            src, dst = dst, src

    def plain():
        ctx.enqueue_batched(dt, G.ADD, G.MIN, d.data_ptr(), d.data_ptr(), tmp.data_ptr(), n, n, n, batch, stream=s)

    torch.cuda.synchronize()
    closure()
    squaring()   # ceil(log2 N) squarings cover every path of up to 2^ceil(log2 N) >= N edges: the fixed point
    torch.cuda.synchronize()
    last = x if squarings % 2 == 0 else y
    identical = bool(torch.equal(d.view(torch.int32), last.view(torch.int32)))
    for fn in (closure, squaring, plain):   # warm-up
        fn()
    torch.cuda.synchronize()
    times = {"closure": [], "squaring": [], "plain": []}
    for _ in range(rounds):
        for arm, fn in (("closure", closure), ("squaring", squaring), ("plain", plain)):
            times[arm].append(window(fn, seconds))
    med = {arm: statistics.median(v) for arm, v in times.items()}

    # per-phase kernel time of one call, in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        closure()
        torch.cuda.synchronize()
    split = {p: 0.0 for p, _ in PHASES}
    for ev in prof.key_averages():
        for p, kname in PHASES:
            if kname in ev.key:
                split[p] += ev.device_time_total / 1000.0   # us -> ms
    return {"workload": name, "n": n, "batch": batch, "squarings": squarings, "ms": med, "windows_ms": times,
            "closure_over_plain": med["closure"] / med["plain"], "squaring_over_closure": med["squaring"] / med["closure"],
            "closure_equals_squaring": identical, "profiled_phase_ms": split}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workload", nargs="*", default=list(WORKLOADS))
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_closure.py needs a CUDA device")
    name, power, clock = gpu_info()
    print("GPU: %s, power limit %s, max SM clock %s" % (name, power, clock))
    results = []
    with G.Context(0) as ctx, torch.cuda.stream(torch.cuda.Stream()):
        for w in args.workload:
            r = bench(ctx, w, args.seconds, args.rounds)
            results.append(r)
            ph = r["profiled_phase_ms"]
            print("%-24s closure %9.3f ms  squaring %9.3f ms  plain %9.3f ms  closure/plain %.3f  squaring/closure "
                  "%.2f  identical %s  phases: pivot %.3f panel %.3f remainder %.3f ms" % (
                      w, r["ms"]["closure"], r["ms"]["squaring"], r["ms"]["plain"], r["closure_over_plain"],
                      r["squaring_over_closure"], r["closure_equals_squaring"], ph["pivot"], ph["panel"],
                      ph["remainder"]), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit": power, "max_sm_clock": clock, "results": results}, f, indent=1)
    if not all(r["closure_equals_squaring"] for r in results):
        sys.exit("the closure and repeated squaring wrote different bytes")


if __name__ == "__main__":
    main()
