#!/usr/bin/env python
"""The accumulating call (mm_kernel_enqueue_accumulate) against the workaround it replaces, on one GPU.

    python scripts/bench_accumulate.py [--seconds 1.0] [--rounds 3] [--workload NAME ...] [--json FILE]

Three arms per workload, on the same device buffers:
  acc     enqueue_accumulate: C <- C (+) A (x) B in the compute kernel's epilogue
  split   the plain call into a temporary, then the same R on the device with torch (float / half add,
          torch.minimum on the NaN-free data used here)
  plain   the plain call alone (writes C, reads nothing of it)
Workloads: float 16384^3, float 16384 x 512 x 16384 (a rank-512 update, where C's traffic is comparable to the
arithmetic), float (Add, Min) 8192 x 256 x 8192 (one blocked shortest-path relaxation), half 16384 x 1024 x 16384.
Each arm is warmed up, then the arms are timed alternately, `--rounds` windows each of at least `--seconds` of device
work (CUDA events); the median window is reported as milliseconds per call.  In every run the acc and split arms must
have written identical bytes (checked once, from the same C_old).  The card's name, power limit and SM clock limit are
read in the same run.  Needs a CUDA device; no fallback.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import gemm_hls_b200 as G  # noqa: E402

# name: (dtype, map, reduce, N, K, M)
WORKLOADS = {
    "float_16384": (G.FLOAT, G.MULTIPLY, G.ADD, 16384, 16384, 16384),
    "float_rank512": (G.FLOAT, G.MULTIPLY, G.ADD, 16384, 512, 16384),
    "float_addmin_8192x256": (G.FLOAT, G.ADD, G.MIN, 8192, 256, 8192),
    "half_16384x1024": (G.HALF, G.MULTIPLY, G.ADD, 16384, 1024, 16384),
}
TORCH_DTYPE = {G.FLOAT: torch.float32, G.HALF: torch.float16}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, clock = [x.strip() for x in out.split(",")]
    return name, power, clock


def window(fn, seconds):
    """ms per call over a window of at least `seconds` of device time (the call count grows at most tenfold per try)."""
    calls = 1
    while True:
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(calls):
            fn()
        stop.record()
        stop.synchronize()
        ms = start.elapsed_time(stop)
        if ms >= 1000.0 * seconds:
            return ms / calls
        calls = min(10 * calls, max(2 * calls, int(calls * 1200.0 * seconds / max(ms, 1e-3)) + 1))


def bench(ctx, name, seconds, rounds):
    dt, mp, rd, n, k, m = WORKLOADS[name]
    tdt = TORCH_DTYPE[dt]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    scale = 1.0 if dt == G.FLOAT else 0.05          # half: keep sums far from the overflow threshold
    a = ((torch.rand((n, k), generator=gen, device="cuda") * 9 + 1) * scale).to(tdt)
    b = ((torch.rand((k, m), generator=gen, device="cuda") * 9 + 1) * scale).to(tdt)
    c0 = (torch.rand((n, m), generator=gen, device="cuda") * 100 + 1).to(tdt)
    c_acc, c_split, tmp = c0.clone(), c0.clone(), torch.empty_like(c0)
    s = torch.cuda.current_stream().cuda_stream
    reduce_ = torch.add if rd == G.ADD else torch.minimum

    def acc():
        ctx.enqueue_accumulate(dt, mp, rd, a.data_ptr(), b.data_ptr(), c_acc.data_ptr(), n, k, m, stream=s)

    def split():
        ctx.enqueue(dt, mp, rd, a.data_ptr(), b.data_ptr(), tmp.data_ptr(), n, k, m, stream=s)
        reduce_(c_split, tmp, out=c_split)

    def plain():
        ctx.enqueue(dt, mp, rd, a.data_ptr(), b.data_ptr(), tmp.data_ptr(), n, k, m, stream=s)

    torch.cuda.synchronize()
    acc()
    split()
    torch.cuda.synchronize()
    ibits = torch.int32 if dt == G.FLOAT else torch.int16
    identical = bool(torch.equal(c_acc.view(ibits), c_split.view(ibits)))
    for fn in (acc, split, plain):   # warm-up
        fn()
    torch.cuda.synchronize()
    times = {"acc": [], "split": [], "plain": []}
    for _ in range(rounds):
        for arm, fn in (("acc", acc), ("split", split), ("plain", plain)):
            times[arm].append(window(fn, seconds))
    med = {arm: statistics.median(v) for arm, v in times.items()}
    return {"workload": name, "n": n, "k": k, "m": m, "ms": med, "windows_ms": times,
            "acc_over_plain": med["acc"] / med["plain"], "split_over_acc": med["split"] / med["acc"],
            "acc_equals_split": identical}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workload", nargs="*", default=list(WORKLOADS))
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_accumulate.py needs a CUDA device")
    name, power, clock = gpu_info()
    print("GPU: %s, power limit %s, max SM clock %s" % (name, power, clock))
    results = []
    # one non-default stream for the library calls, torch's reductions and the events (the legacy default stream would
    # make the library fall back to its own stream, which does not order with torch's)
    with G.Context(0) as ctx, torch.cuda.stream(torch.cuda.Stream()):
        for w in args.workload:
            r = bench(ctx, w, args.seconds, args.rounds)
            results.append(r)
            print("%-22s acc %8.3f ms  split %8.3f ms  plain %8.3f ms  acc/plain %.3f  split/acc %.3f  identical %s" % (
                w, r["ms"]["acc"], r["ms"]["split"], r["ms"]["plain"], r["acc_over_plain"], r["split_over_acc"],
                r["acc_equals_split"]), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit": power, "max_sm_clock": clock, "results": results}, f, indent=1)
    if not all(r["acc_equals_split"] for r in results):
        sys.exit("the accumulate call and the workaround wrote different bytes")


if __name__ == "__main__":
    main()
