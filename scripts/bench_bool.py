#!/usr/bin/env python
"""Bit-packed Boolean products and closures (mm_kernel_enqueue_bool / _closure) against the uint8 (And, Max) semiring
calls they replace, on one GPU.

    python scripts/bench_bool.py [--seconds 1.0] [--rounds 3] [--json FILE]

  (i)   product 16384^3: enqueue_bool on packed bits vs the uint8 (And, Max) product on the same graph unpacked;
  (ii)  closure at N = 16384 and 32768: enqueue_bool_closure vs the uint8 (And, Max) closure (at 32768 the uint8 arm
        runs once, untimed windows being too long);
  (iii) the closure vs repeated squaring D <- D | D.D through enqueue_bool, to the fixed point (the count of squarings
        is found once on the data, then timed).
Each pair of arms must write identical bits after packing (checked once per workload).  Arms are warmed up and timed
alternately, `--rounds` windows each of at least `--seconds` of device work (CUDA events); the median is reported.
Then one call of each Boolean arm runs under torch.profiler for kernel and phase times.  Rates are 2 N K M bit
operations over kernel time; the closure's phase 3 is also given as its D traffic (it reads and writes D once per
round: 2 (N - 256)^2 / 8 bytes) over its time, as a share of the H100 SXM's 3.35 TB/s.  The b1 tensor cores have no
data-sheet peak, so no tensor share of peak is claimed.  The card's name and power limit are read in the same run.
Needs a CUDA device; no fallback.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402
import gemm_hls_b200 as G  # noqa: E402
from bench_accumulate import gpu_info, window  # noqa: E402

HBM = 3.35e12
B = 256   # the closure's block of indices (DESIGN.md 3.10)
WEIGHTS = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8)


def pack(x):
    """0/1 uint8 (..., L) on the device -> (..., L / 8) bytes, bit j % 8 of byte j / 8 (numpy.packbits 'little')."""
    w = WEIGHTS.to(x.device)
    return (x.view(*x.shape[:-1], -1, 8) * w).sum(-1, dtype=torch.uint8)


def unpack(p):
    w = WEIGHTS.to(p.device)
    return ((p.unsqueeze(-1) & w) != 0).to(torch.uint8).view(*p.shape[:-1], -1)


def random_bits(n, m, density, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return (torch.rand((n, m), generator=g, device="cuda") < density).to(torch.uint8)


def profiled(fn, names):
    """Device ms of one fn() per kernel-name fragment, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in names}
    for ev in prof.key_averages():
        for k, frag in names.items():
            if frag in ev.key:
                out[k] += ev.device_time_total / 1000.0
    return out


def timed(arms, seconds, rounds):
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a, fn in arms.items():
            times[a].append(window(fn, seconds))
    return {a: statistics.median(v) for a, v in times.items()}, times


def product_workload(ctx, s, n, seconds, rounds):
    a8, b8 = random_bits(n, n, 1.0 / 64, 1), random_bits(n, n, 1.0 / 64, 2)
    a, b = pack(a8), pack(b8)
    c, c8 = torch.empty_like(a), torch.empty_like(a8)
    arms = {"bool": lambda: ctx.enqueue_bool(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, n, n, stream=s),
            "uint8_and_max": lambda: ctx.enqueue(G.UINT8, G.AND, G.MAX, a8.data_ptr(), b8.data_ptr(), c8.data_ptr(),
                                                 n, n, n, stream=s)}
    arms["bool"]()
    arms["uint8_and_max"]()
    torch.cuda.synchronize()
    identical = bool(torch.equal(c, pack(c8)))
    ones = float(unpack(c).float().mean())
    med, win = timed(arms, seconds, rounds)
    k = profiled(arms["bool"], {"transpose": "bit_transpose_kernel", "gemm": "gemm_wgmma_kernel"})
    ops = 2.0 * n ** 3
    return {"workload": "product_%d" % n, "ms": med, "windows_ms": win, "identical": identical, "ones": ones,
            "kernel_ms": k, "bool_tops_kernel": ops / (k["gemm"] * 1e-3) / 1e12,
            "bool_tops_call": ops / (med["bool"] * 1e-3) / 1e12,
            "uint8_tops_call": ops / (med["uint8_and_max"] * 1e-3) / 1e12,
            "uint8_over_bool": med["uint8_and_max"] / med["bool"]}


def closure_workload(ctx, s, n, seconds, rounds, uint8_once):
    d8 = random_bits(n, n, 2.0 / n, 3)
    d = pack(d8)
    x, tmp, xs, ys = d.clone(), torch.empty_like(d8), d.clone(), torch.empty_like(d)
    res = {"workload": "closure_%d" % n}

    def closure():
        x.copy_(d)
        ctx.enqueue_bool_closure(x.data_ptr(), n, stream=s)

    def uint8_closure():
        tmp.copy_(d8)
        ctx.enqueue_closure(G.UINT8, G.AND, G.MAX, tmp.data_ptr(), n, stream=s)

    # squaring: the count needed for the fixed point, found once
    xs.copy_(d)
    squarings = 0
    while True:
        ctx.enqueue_bool(xs.data_ptr(), xs.data_ptr(), ys.data_ptr(), n, n, n, stream=s)
        ys |= xs
        squarings += 1
        if torch.equal(xs, ys):
            break
        xs.copy_(ys)

    def squaring():
        xs.copy_(d)
        for _ in range(squarings):
            ctx.enqueue_bool(xs.data_ptr(), xs.data_ptr(), ys.data_ptr(), n, n, n, stream=s)
            torch.bitwise_or(ys, xs, out=xs)

    closure()
    uint8_closure()
    torch.cuda.synchronize()
    res["identical_uint8"] = bool(torch.equal(x, pack(tmp)))
    res["identical_squaring"] = bool(torch.equal(x, ys))
    res["ones"] = float(unpack(x).float().mean())
    res["squarings"] = squarings
    arms = {"closure": closure, "squaring": squaring}
    if uint8_once:
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        uint8_closure()
        stop.record()
        stop.synchronize()
        res["uint8_closure_ms_once"] = start.elapsed_time(stop)
    else:
        arms["uint8_closure"] = uint8_closure
    res["ms"], res["windows_ms"] = timed(arms, seconds, rounds)
    u8 = res["ms"].get("uint8_closure", res.get("uint8_closure_ms_once"))
    res["uint8_over_closure"] = u8 / res["ms"]["closure"]
    res["squaring_over_closure"] = res["ms"]["squaring"] / res["ms"]["closure"]
    k = profiled(lambda: ctx.enqueue_bool_closure(x.data_ptr(), n, stream=s),
                 {"diagonal": "closure_diagonal_kernel", "panels": "closure_tile_kernel<true>",
                  "remainder": "closure_tile_kernel<false>"})
    res["phase_ms"] = k
    rounds_ = (n + B - 1) // B
    res["tops_kernel"] = 2.0 * n ** 3 / (sum(k.values()) * 1e-3) / 1e12
    p3_bytes = rounds_ * 2.0 * (n - B) ** 2 / 8
    res["phase3_tb_s"] = p3_bytes / (k["remainder"] * 1e-3) / 1e12
    res["phase3_hbm_share"] = p3_bytes / (k["remainder"] * 1e-3) / HBM
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--product-n", type=int, default=16384)
    ap.add_argument("--closure-n", type=int, nargs="*", default=[16384, 32768])
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_bool.py needs a CUDA device")
    name, power, clock = gpu_info()
    print("GPU: %s, power limit %s, max SM clock %s" % (name, power, clock), flush=True)
    results = []
    with G.Context(0) as ctx, torch.cuda.stream(torch.cuda.Stream()):
        s = torch.cuda.current_stream().cuda_stream
        r = product_workload(ctx, s, args.product_n, args.seconds, args.rounds)
        results.append(r)
        print("product %d^3: bool %.3f ms (gemm %.3f + transpose %.3f ms kernel, %.1f T bit-op/s kernel)  uint8 (And, "
              "Max) %.3f ms  uint8/bool %.1f  identical %s" % (
                  args.product_n, r["ms"]["bool"], r["kernel_ms"]["gemm"], r["kernel_ms"]["transpose"],
                  r["bool_tops_kernel"], r["ms"]["uint8_and_max"], r["uint8_over_bool"], r["identical"]), flush=True)
        for n in args.closure_n:
            r = closure_workload(ctx, s, n, args.seconds, args.rounds, uint8_once=n >= 32768)
            results.append(r)
            ph = r["phase_ms"]
            print("closure %d: bool %.3f ms  uint8 %.3f ms%s  squaring (%d) %.3f ms  uint8/bool %.1f  squaring/bool "
                  "%.2f  identical uint8 %s squaring %s  phases: diagonal %.3f panels %.3f remainder %.3f ms "
                  "(%.2f TB/s, %.0f%% of 3.35 TB/s)" % (
                      n, r["ms"]["closure"], r["ms"].get("uint8_closure", r.get("uint8_closure_ms_once")),
                      " (once)" if "uint8_closure_ms_once" in r else "", r["squarings"], r["ms"]["squaring"],
                      r["uint8_over_closure"], r["squaring_over_closure"], r["identical_uint8"],
                      r["identical_squaring"], ph["diagonal"], ph["panels"], ph["remainder"], r["phase3_tb_s"],
                      100 * r["phase3_hbm_share"]), flush=True)
    out = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "results": results}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit": power, "identical": all(
        r.get("identical", True) and r.get("identical_uint8", True) and r.get("identical_squaring", True)
        for r in results)}))
    if not all(r.get("identical", True) and r.get("identical_uint8", True) and r.get("identical_squaring", True)
               for r in results):
        sys.exit("the arms wrote different bits")


if __name__ == "__main__":
    main()
