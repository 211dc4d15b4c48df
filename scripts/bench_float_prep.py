#!/usr/bin/env python
"""Float operand preparation at 16384^3 on the three kinds of data that decide what it writes.

    python scripts/bench_float_prep.py [--n 16384] [--steps 10] [--warmup 3] [--profile DIR]

  fit     U[1, 10) (bench.py's data): every operand fits in half, the f16 datapath
  early   N(0, 1) with B[0, 0] = 1e-6: the first item does not fit, the rest settles on TF32
  late    U[1, 10) with A[N-1, K-1] = 2^17: only the last item does not fit (the worst case for preparation)

Each kind runs `steps` calls through ctx.enqueue with the context's profiling on, after `warmup` calls, and prints one
JSON line per kind: preparation (first event to the GEMM's start), GEMM and step times per call in ms, from CUDA
events.  Two builds are compared by running this script from each tree in turn.  --profile DIR: instead, one
torch.profiler run per kind; prints the mean time of every kernel (the preparation passes by name) and writes the
traces under DIR.  Prints the GPU's name and power limit first.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_line():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out


def operands(torch, kind, n, gen):
    if kind == "early":
        a = torch.randn((n, n), device="cuda", generator=gen)
        b = torch.randn((n, n), device="cuda", generator=gen)
        b[0, 0] = 1e-6
    else:
        a = torch.rand((n, n), device="cuda", generator=gen) * 9 + 1
        b = torch.rand((n, n), device="cuda", generator=gen) * 9 + 1
        if kind == "late":
            a[n - 1, n - 1] = 2.0 ** 17
    return a, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kinds", default="fit,early,late")
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    import torch
    import gemm_hls_b200 as G

    print(json.dumps({"gpu": gpu_line()}), flush=True)
    n = args.n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(0)
    stream = torch.cuda.Stream()   # a stream of its own: handle 0 would select the context's stream
    with G.Context(0) as ctx:
        for kind in args.kinds.split(","):
            a, b = operands(torch, kind, n, gen)
            c = torch.empty((n, n), device="cuda")
            torch.cuda.synchronize()

            def call():
                ctx.enqueue(G.FLOAT, G.MULTIPLY, G.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, n, n,
                            stream=stream.cuda_stream)
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            if args.profile:
                from torch.autograd import DeviceType
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        call()
                    torch.cuda.synchronize()
                os.makedirs(args.profile, exist_ok=True)
                prof.export_chrome_trace(os.path.join(args.profile, "float_prep_%s.json" % kind))
                times = {}
                for e in prof.events():
                    if e.device_type == DeviceType.CUDA:
                        name = re.sub(r"\(anonymous namespace\)::|^void |<.*|\(.*", "", e.name).strip()
                        times.setdefault(name, []).append(e.device_time * 1e-3)
                print(json.dumps({"kind": kind, "kernel_ms_per_call": {name: round(sum(v) / args.steps, 4)
                                                                       for name, v in times.items()}}), flush=True)
                continue
            ctx.set_profiling(True)
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(stream)
            for _ in range(args.steps):
                call()
            ev1.record(stream)
            torch.cuda.synchronize()
            prep_s, main_s, calls = ctx.profile_read()
            ctx.set_profiling(False)
            calls = max(calls, 1)
            print(json.dumps({"kind": kind, "n": n, "steps": args.steps, "prep_ms": round(1e3 * prep_s / calls, 3),
                              "gemm_ms": round(1e3 * main_s / calls, 3),
                              "step_ms": round(ev0.elapsed_time(ev1) / args.steps, 3)}), flush=True)


if __name__ == "__main__":
    main()
