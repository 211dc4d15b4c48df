#!/usr/bin/env python
"""Throughput of one batched call against a loop of single calls, on one GPU.

    python scripts/bench_batched.py [--seconds 1.0] [--rounds 3] [--workload NAME ...] [--json FILE]

For each workload, both arms run on the same stream and the same device buffers:
  * batched: one mm_kernel_enqueue_batched over the whole batch;
  * loop:    `batch` mm_kernel_enqueue calls, one per problem.
Both arms are warmed up, then timed alternately (`--rounds` times each) with CUDA events over a window of
at least `--seconds` of device work.  The script reports the median rate of each arm in GFLOP/s (2 N K M
operations per problem; GOp/s for a semiring) and their ratio, and checks that the two arms wrote the
same bytes.  The card's name and power limit are read in the same run and printed with the numbers.
Needs a CUDA device; there is no fallback.
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

# name: (dtype, map, reduce, flags, batch, n, k, m)
WORKLOADS = {
    "float_64x512": (G.FLOAT, G.MULTIPLY, G.ADD, 0, 64, 512, 512, 512),
    "half_64x512": (G.HALF, G.MULTIPLY, G.ADD, 0, 64, 512, 512, 512),
    "uint8_64x512": (G.UINT8, G.MULTIPLY, G.ADD, 0, 64, 512, 512, 512),
    "double_64x256": (G.DOUBLE, G.MULTIPLY, G.ADD, 0, 64, 256, 256, 256),
    "addmin_64x513x528x528": (G.FLOAT, G.ADD, G.MIN, 0, 64, 513, 528, 528),
    "float_64x512_shared_b": (G.FLOAT, G.MULTIPLY, G.ADD, G.FLAG_BATCH_SHARED_B, 64, 512, 512, 512),
}
TORCH_DTYPE = {G.FLOAT: torch.float32, G.HALF: torch.float16, G.DOUBLE: torch.float64, G.UINT8: torch.uint8}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def operands(dtype, shape, gen):
    if dtype == G.UINT8:
        return torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)
    x = torch.rand(shape, dtype=torch.float32, device="cuda", generator=gen) * 9 + 1   # U[1, 10], like the reference
    return x.to(TORCH_DTYPE[dtype])


def run(ctx, name, stream, seconds, rounds):
    dtype, mp, rd, flags, batch, n, k, m = WORKLOADS[name]
    shared_b = bool(flags & G.FLAG_BATCH_SHARED_B)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    a = operands(dtype, (batch, n * k), gen)
    b = operands(dtype, (1 if shared_b else batch, k * m), gen)
    c_batched = torch.zeros((batch, n * m), dtype=a.dtype, device="cuda")
    c_loop = torch.ones((batch, n * m), dtype=a.dtype, device="cuda")
    s = stream.cuda_stream
    single_flags = flags & ~(G.FLAG_BATCH_SHARED_A | G.FLAG_BATCH_SHARED_B)

    def batched():
        ctx.enqueue_batched(dtype, mp, rd, a.data_ptr(), b.data_ptr(), c_batched.data_ptr(), n, k, m, batch,
                            flags=flags, stream=s)

    def loop():
        for i in range(batch):
            ctx.enqueue(dtype, mp, rd, a[i].data_ptr(), b[0 if shared_b else i].data_ptr(), c_loop[i].data_ptr(),
                        n, k, m, flags=single_flags, stream=s)

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    for fn in (batched, loop):   # warm-up: scratch sizes, module loading, clocks
        timed(fn, 3)
    reps = {fn: max(1, int(seconds / timed(fn, 3)) + 1) for fn in (batched, loop)}
    times = {batched: [], loop: []}
    for _ in range(rounds):      # alternate the arms
        for fn in (batched, loop):
            times[fn].append(timed(fn, reps[fn]))
    stream.synchronize()
    identical = torch.equal(c_batched.view(-1).view(torch.uint8), c_loop.view(-1).view(torch.uint8))
    ops = 2.0 * batch * n * k * m
    t_b, t_l = statistics.median(times[batched]), statistics.median(times[loop])
    return {
        "workload": name, "batch": batch, "n": n, "k": k, "m": m,
        "unit": "GFLOP/s" if (mp, rd) == (G.MULTIPLY, G.ADD) else "GOp/s",
        "batched_rate": ops / t_b * 1e-9, "loop_rate": ops / t_l * 1e-9, "speedup": t_l / t_b,
        "batched_seconds": times[batched], "loop_seconds": times[loop],
        "reps": [reps[batched], reps[loop]], "identical": identical,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="minimum device time per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per arm, alternating")
    ap.add_argument("--workload", nargs="*", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batched.py needs a CUDA device")
    card, power = gpu_info()
    print("# %s, power limit %s" % (card, power), flush=True)
    results = []
    stream = torch.cuda.Stream()
    with G.Context(0) as ctx, torch.cuda.stream(stream):
        for name in args.workload:
            r = run(ctx, name, stream, args.seconds, args.rounds)
            r.update(gpu=card, power_limit=power)
            results.append(r)
            print("%-24s batch %3d  batched %9.1f %s  loop %9.1f %s  x%.2f  outputs %s" % (
                name, r["batch"], r["batched_rate"], r["unit"], r["loop_rate"], r["unit"], r["speedup"],
                "identical" if r["identical"] else "DIFFER"), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)
    sys.exit(0 if all(r["identical"] for r in results) else 1)


if __name__ == "__main__":
    main()
