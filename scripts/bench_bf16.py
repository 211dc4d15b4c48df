#!/usr/bin/env python
"""bfloat16 against half on the wgmma GEMM, with torch.matmul in bfloat16 as an outside yardstick, on one GPU.

    python scripts/bench_bf16.py [--sizes 16384 32768] [--seconds 1.0] [--rounds 3] [--json FILE]

For each size S (an S x S x S (Multiply, Add) product) three arms run on the same stream:
  * bf16:  mm_kernel_enqueue with MM_DTYPE_BFLOAT16 (B's K-major copy + the bf16 wgmma GEMM);
  * half:  the same call with MM_DTYPE_HALF on the same values converted to half;
  * torch: torch.matmul in bfloat16, with allow_bf16_reduced_precision_reduction = False.
Each arm is warmed up, then the arms are timed alternately (`--rounds` windows each) with CUDA events over
at least `--seconds` of device work per window; the median window gives the step time.  The library arms'
GEMM kernel time comes from the library's own per-phase events (mm_context_set_profiling) in the same
windows.  The inputs are U[0.5, 1), the same values for every arm.  Rates are 2 S^3 / time.  The bf16
result is checked on a seeded sample of rows against an FP64 evaluation of the same bf16 inputs: every
element within 1 bf16 ulp.  The card's name and power limit are
read in the same run and printed with the numbers.  Needs a CUDA device; there is no fallback.
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, stream, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps


def max_ulps_fp64(c, a, b, rows):
    """Largest |C - A*B| over the sampled rows, in bf16 ulps at the exact result's binade."""
    ref = a[rows].double() @ b.double()
    ulp = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126))) - 7)
    return ((c[rows].double() - ref).abs() / ulp).max().item()


def run(ctx, size, stream, seconds, rounds):
    n = k = m = size
    s = stream.cuda_stream
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    # U[0.5, 1): same-sign data (nothing cancels, so the 1-ulp check is meaningful), and C = O(K) stays inside half's
    # range at 32768^3.  Every bf16 value in [0.5, 1) is exact in half: both arms multiply the same numbers.
    a = (torch.rand((n, k), device="cuda", generator=gen) * 0.5 + 0.5).to(torch.bfloat16)
    b = (torch.rand((k, m), device="cuda", generator=gen) * 0.5 + 0.5).to(torch.bfloat16)
    ah, bh = a.to(torch.float16), b.to(torch.float16)
    c_bf = torch.empty((n, m), dtype=torch.bfloat16, device="cuda")
    c_h = torch.empty((n, m), dtype=torch.float16, device="cuda")
    c_t = torch.empty((n, m), dtype=torch.bfloat16, device="cuda")
    arms = {
        "bf16": lambda: ctx.enqueue(G.BFLOAT16, G.MULTIPLY, G.ADD, a.data_ptr(), b.data_ptr(), c_bf.data_ptr(),
                                    n, k, m, stream=s),
        "half": lambda: ctx.enqueue(G.HALF, G.MULTIPLY, G.ADD, ah.data_ptr(), bh.data_ptr(), c_h.data_ptr(),
                                    n, k, m, stream=s),
        "torch_bf16": lambda: torch.matmul(a, b, out=c_t),
    }
    for fn in arms.values():   # warm-up: scratch sizes, module loading, algorithm selection, clocks
        timed(fn, stream, 2)
    reps = {name: min(256, max(1, int(seconds / timed(fn, stream, 2)) + 1)) for name, fn in arms.items()}
    times = {name: [] for name in arms}
    kernels = {"bf16": [], "half": []}
    for _ in range(rounds):    # alternate the arms
        for name, fn in arms.items():
            if name in kernels:   # the GEMM kernel alone, from the library's per-phase events in the same window
                ctx.set_profiling(True)
            times[name].append(timed(fn, stream, reps[name]))
            if name in kernels:
                _, main, calls = ctx.profile_read()
                ctx.set_profiling(False)
                kernels[name].append(main / calls)
    kernel = {name: statistics.median(v) for name, v in kernels.items()}
    stream.synchronize()
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    rows = torch.randint(0, n, (64,), device="cuda", generator=g)
    ulps = max_ulps_fp64(c_bf, a, b, rows)
    flops = 2.0 * n * k * m
    out = {"size": size, "reps": reps, "max_ulps_vs_fp64": ulps, "finite": bool(torch.isfinite(c_bf).all())}
    for name in arms:
        step = statistics.median(times[name])
        out[name] = {"step_s": step, "step_tflops": flops / step * 1e-12, "windows_s": times[name]}
        if name in kernel:
            out[name].update(kernel_s=kernel[name], kernel_tflops=flops / kernel[name] * 1e-12)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[16384, 32768])
    ap.add_argument("--seconds", type=float, default=1.0, help="minimum device time per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per arm, alternating")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_bf16.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    card, power = gpu_info()
    print("# %s, power limit %s" % (card, power), flush=True)
    results = []
    stream = torch.cuda.Stream()
    with G.Context(0) as ctx, torch.cuda.stream(stream):
        for size in args.sizes:
            r = run(ctx, size, stream, args.seconds, args.rounds)
            r.update(gpu=card, power_limit=power)
            results.append(r)
            line = "%6d^3" % size
            for name in ("bf16", "half", "torch_bf16"):
                x = r[name]
                line += "  %s step %.2f ms %.0f TFLOP/s" % (name, 1e3 * x["step_s"], x["step_tflops"])
                if "kernel_s" in x:
                    line += " (kernel %.2f ms %.0f)" % (1e3 * x["kernel_s"], x["kernel_tflops"])
            line += "  bf16 vs fp64: %.3f ulp max" % r["max_ulps_vs_fp64"]
            print(line, flush=True)
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)
    sys.exit(0 if all(r["max_ulps_vs_fp64"] <= 1.0 and r["finite"] for r in results) else 1)


if __name__ == "__main__":
    main()
