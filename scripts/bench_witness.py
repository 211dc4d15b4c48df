#!/usr/bin/env python
"""Throughput of the witness call (mm_kernel_enqueue_witness) against the plain call, on one GPU.

    python scripts/bench_witness.py [--seconds 1.0] [--rounds 3] [--workload NAME ...] [--json FILE]

Workloads: float (Add, Min) 8192^3 at flags 0 (FMNMX) and under MM_FLAG_EXACT, int32 (Add, Max) 8192^3.  Both arms
use the same device buffers for A, B and C; they are warmed up, then timed alternately (`--rounds` windows each) with
CUDA events over at least `--seconds` of device work.  Reported per arm: the median rate in TOp/s at 2 N K M
operations, the ratio witness / plain, and the share of the derived issue ceiling of the kernel that ran:
132 SMs x 4 schedulers x 32 lanes x the SM clock / (issue slots per element-step), at 2 operations per element-step.
The slots are counted in the kernel's SASS (instructions of the unrolled main loop / element-steps of one k-tile),
the way DESIGN.md section 3.6 derives 33.5 TOp/s for the plain kernel.  The two arms' C must be byte-identical.
The card's name, power limit and SM clock limit are read in the same run.  Needs a CUDA device; no fallback.
"""
import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import gemm_hls_b200 as G  # noqa: E402

# name: (dtype, map, reduce, flags, object, kernel tags (Map, Reduce) in the mangled names)
WORKLOADS = {
    "float_addmin_8192": (G.FLOAT, G.ADD, G.MIN, 0, "f32_1", ("3Sum", "7MinFast")),
    "float_addmin_8192_exact": (G.FLOAT, G.ADD, G.MIN, G.FLAG_EXACT, "f32_1", ("3Sum", "3Min")),
    "int32_addmax_8192": (G.INT32, G.ADD, G.MAX, 0, "i32_1", ("3Sum", "3Max")),
}
N = K = M = 8192
SMS, SCHEDULERS, LANES = 132, 4, 32
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
    except Exception:
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return name, power, clock


def issue_slots(obj, kernel, tags):
    """Issue slots per element-step of `kernel` (the ring variant: one k-tile of 16 k x 8 x 8 elements = 1024
    element-steps per thread, fully unrolled): the instructions from the first to the last one of the opcodes that
    occur once per element-step (1000 times or more), loads and address arithmetic between them included, over 1024."""
    path = os.path.join(ROOT, "gemm_hls_b200", "build", obj)
    if not os.path.exists(path):
        return None
    text = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True).stdout
    ops, name = [], None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][^;\s]*)", line)
        if m and name and kernel + "I" in name and re.search(r"I\w(?:NS_)?%s.*%s" % tags, name):
            ops.append(m.group(1))
    per_step = {op for op in set(ops) if ops.count(op) >= 1000}
    idx = [i for i, op in enumerate(ops) if op in per_step]
    return (idx[-1] - idx[0] + 1) / 1024.0 if idx else None


def run(ctx, name, stream, seconds, rounds):
    dtype, mp, rd, flags, _, _ = WORKLOADS[name]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    if dtype == G.FLOAT:
        a = torch.rand((N, K), generator=gen, device="cuda") * 9 + 1
        b = torch.rand((K, M), generator=gen, device="cuda") * 9 + 1
    else:
        a = torch.randint(-2 ** 20, 2 ** 20, (N, K), generator=gen, device="cuda", dtype=torch.int32)
        b = torch.randint(-2 ** 20, 2 ** 20, (K, M), generator=gen, device="cuda", dtype=torch.int32)
    c_plain = torch.zeros((N, M), dtype=a.dtype, device="cuda")
    c_wit = torch.ones((N, M), dtype=a.dtype, device="cuda")
    w = torch.empty((N, M), dtype=torch.int32, device="cuda")
    s = stream.cuda_stream

    def plain():
        ctx.enqueue(dtype, mp, rd, a.data_ptr(), b.data_ptr(), c_plain.data_ptr(), N, K, M, flags=flags, stream=s)

    def witness():
        ctx.enqueue_witness(dtype, mp, rd, a.data_ptr(), b.data_ptr(), c_wit.data_ptr(), w.data_ptr(), N, K, M,
                            flags=flags, stream=s)

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    for fn in (plain, witness):
        timed(fn, 2)
    reps = {fn: max(1, int(seconds / timed(fn, 2)) + 1) for fn in (plain, witness)}
    times = {plain: [], witness: []}
    for _ in range(rounds):
        for fn in (plain, witness):
            times[fn].append(timed(fn, reps[fn]))
    stream.synchronize()
    identical = torch.equal(c_plain.view(torch.int32), c_wit.view(torch.int32))
    ops = 2.0 * N * K * M
    tp, tw = statistics.median(times[plain]), statistics.median(times[witness])
    return {"workload": name, "n": N, "k": K, "m": M, "flags": flags,
            "plain_tops": ops / tp * 1e-12, "witness_tops": ops / tw * 1e-12, "ratio": tp / tw,
            "plain_seconds": times[plain], "witness_seconds": times[witness], "reps": [reps[plain], reps[witness]],
            "identical": identical}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="minimum device time per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per arm, alternating")
    ap.add_argument("--workload", nargs="*", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_witness.py needs a CUDA device")
    card, power, clock = gpu_info()
    print("# %s, power limit %s, max SM clock %s" % (card, power, clock), flush=True)
    mhz = float(clock.split()[0]) if clock.split()[0].replace(".", "").isdigit() else None
    results = []
    stream = torch.cuda.Stream()
    with G.Context(0) as ctx, torch.cuda.stream(stream):
        for name in args.workload:
            r = run(ctx, name, stream, args.seconds, args.rounds)
            _, _, _, _, obj, tags = WORKLOADS[name]
            for arm, obj_name, kernel in (("plain", "semiring_%s.o" % obj, "semiring_ring_kernel"),
                                          ("witness", "semiring_witness_%s.o" % obj, "semiring_witness_ring_kernel")):
                slots = issue_slots(obj_name, kernel, tags)
                r[arm + "_slots_per_step"] = slots
                if slots and mhz:
                    ceiling = SMS * SCHEDULERS * LANES * mhz * 1e6 / slots * 2 * 1e-12
                    r[arm + "_ceiling_tops"] = ceiling
                    r[arm + "_share"] = r[arm + "_tops"] / ceiling
            r.update(gpu=card, power_limit=power, max_sm_clock=clock)
            results.append(r)
            print("%-26s plain %6.2f TOp/s (%.2f slots/step, %.2f of %.1f)  witness %6.2f TOp/s (%.2f slots/step, "
                  "%.2f of %.1f)  ratio %.3f  C %s" % (
                      name, r["plain_tops"], r.get("plain_slots_per_step") or 0, r.get("plain_share") or 0,
                      r.get("plain_ceiling_tops") or 0, r["witness_tops"], r.get("witness_slots_per_step") or 0,
                      r.get("witness_share") or 0, r.get("witness_ceiling_tops") or 0, r["ratio"],
                      "identical" if r["identical"] else "DIFFERS"), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)
    sys.exit(0 if all(r["identical"] for r in results) else 1)


if __name__ == "__main__":
    main()
