"""Every bench.py workload at its bench size with the default tuning, every element of C against an independent
reference computed on the device, at zero tolerance or bit for bit (run with `-m gpu` on an H100).

At these sizes the kernels run schedules that the test-size suites never reach: at float 16384^3 the wgmma GEMM
runs 4096 tiles of 512 k-blocks on 66 CTA groups (62 or more tiles each, the epilogue's staging reused hundreds of
times per CTA); at half and bf16 32768^3 every operand is 2 GiB, so byte offsets reach 2^31; the (Add, Min) ring
kernel runs 4096 CTAs of 512 k-tiles.  The checks of tests/test_full_size_gpu.py and bench.py sample a few rows.

* Tensor-core paths: exact data (tensor_numerics.full_size_scheme), so the FP64 product is the exact C and the
  output type is reached by one rounding, the epilogue's.  uint8: full-range bytes, the exact sum modulo 256.
* (Add, Min) float and half (Multiply, Add) under MM_FLAG_EXACT: bench.py's data, against Naive<>'s order of
  operations restated in torch on the device (tests/full_size_check.py), bit for bit.
* C and a 4 KiB guard after it are poisoned first (bytes 0xFF, NaN in every float type; uint8 runs with 0x00 and
  0xFF).  The guard must be unchanged.  A mismatch reports the count, the first wrong element and the tile or CTA
  that wrote it.

Each workload is one test that computes its reference once for all its flag and tuning settings, then frees its
tensors, so that the 32768^3 cases fit beside whatever ran before.  On one H100 80GB HBM3 at a 700 W power limit
the file took 24 s, and torch's peak allocation was 16.0 GiB (half and bf16 32768^3; the library's own scratch is
not counted there).
"""
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_size_check as fc  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    props = t.cuda.get_device_properties(0)
    print("full-size exact: %s, %d SMs" % (props.name, props.multi_processor_count))
    return t


@pytest.fixture(autouse=True)
def _release(torch):
    """Report the peak device memory of the test, and hand the cached blocks back when it ends."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print("peak device memory %.1f GiB, %.1f s" % (torch.cuda.max_memory_allocated() / 2.0 ** 30,
                                                   time.perf_counter() - t0))
    torch.cuda.empty_cache()


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _enqueue(torch, mm, ctx, dtype, mp, rd, a, b, torch_dtype, flags=0, poison=0xFF):
    """One mm_kernel_enqueue on a torch stream (bench.py's step()) into a poisoned C with a poisoned guard after it.
    Returns (C, guard)."""
    n, k = a.shape
    m = b.shape[1]
    nbytes = n * m * torch.empty((), dtype=torch_dtype).element_size()
    raw = torch.full((nbytes + fc.GUARD,), poison, dtype=torch.uint8, device="cuda")
    c = raw[:nbytes].view(torch_dtype).view(n, m)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    ctx.enqueue(dtype, mp, rd, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, flags=flags,
                stream=stream.cuda_stream)
    stream.synchronize()
    return c, raw[nbytes:]


def _check(torch, what, c, guard, want, locate, mode, poison):
    fc.check_guard(torch, what, guard, poison)
    fc.compare(torch, what, c, want, locate, mode, poison)


def _run_settings(torch, mm, settings, a, b, want, locate_for, dtype, mp, rd, mode, poisons=(0xFF,)):
    """Each (name, tuning knobs, flags) of `settings` on a fresh context; every failure is collected so that one
    report covers all of them."""
    failures = []
    for name, knobs, flags in settings:
        with mm.Context(0) as ctx:
            ctx.set_tuning(**knobs)
            for poison in poisons:
                what = "%s [poison 0x%02X]" % (name, poison)
                c, guard = _enqueue(torch, mm, ctx, dtype, mp, rd, a, b, want.dtype, flags=flags, poison=poison)
                try:
                    _check(torch, what, c, guard, want, locate_for(knobs), mode, poison)
                    print("%s: every element exact" % what)
                except AssertionError as e:
                    failures.append(str(e))
                del c, guard
    assert not failures, "\n".join(failures)


def _tensor_core_case(torch, mm, path, n, settings, seed, poisons=(0xFF,)):
    a, b = fc.exact_operands(torch, path, n, n, n, seed, "cuda")
    want = fc.fp64_reference(torch, path, a, b)
    dtype = {"tf32": mm.FLOAT, "tf32h": mm.FLOAT, "f16": mm.HALF, "bf16": mm.BFLOAT16, "u8": mm.UINT8,
             "dmma": mm.DOUBLE}[path]
    if path == "dmma":
        sms = _sms(torch)
        locate_for = lambda knobs: fc.grid_locator("gemm_dmma_tma_kernel", fc.dmma_tile_rows(
            n, n, sms, knobs.get("dmma_tile_rows", 0)), fc.DMMA_TILE_COLS, n, n)
    else:
        locate_for = lambda knobs: fc.wgmma_locator(n, n, _sms(torch))
    _run_settings(torch, mm, settings, a, b, want, locate_for, dtype, mm.MULTIPLY, mm.ADD, "value", poisons)


def test_float_16384_tf32_and_3xtf32_exact(torch, mm):
    """bench.py float16384, the headline: data that fits a half, on the f16 datapath of the float wgmma GEMM, and the
    same data under MM_FLAG_TF32X3."""
    assert mm.kernel_path(mm.FLOAT) == "wgmma_tf32"
    _tensor_core_case(torch, mm, "tf32h", 16384, [("float 16384^3 f16 datapath", {}, 0),
                                                  ("float 16384^3 3xtf32", {}, mm.FLAG_TF32X3)], seed=41)


def test_float_16384_tf32_datapath_exact(torch, mm):
    """bench.py float16384 on the TF32 datapath: the same kind of data with A's last row times 2^20, which no half
    holds."""
    _tensor_core_case(torch, mm, "tf32", 16384, [("float 16384^3 tf32 datapath", {}, 0)], seed=41)


def test_half_32768_f16_exact(torch, mm):
    """bench.py half32768: f16 wgmma, 2 GiB operands."""
    assert mm.kernel_path(mm.HALF) == "wgmma_f16"
    _tensor_core_case(torch, mm, "f16", 32768, [("half 32768^3 f16", {}, 0)], seed=42)


def test_bf16_32768_exact(torch, mm):
    """bf16 wgmma at 32768^3 (scripts/bench_bf16.py's largest size)."""
    assert mm.kernel_path(mm.BFLOAT16) == "wgmma_bf16"
    _tensor_core_case(torch, mm, "bf16", 32768, [("bf16 32768^3", {}, 0)], seed=43)


def test_uint8_16384_exact(torch, mm):
    """bench.py uint8_16384: u8 wgmma on full-range bytes, the low byte of the exact sum; poison 0x00 and 0xFF,
    because every byte is a legal result."""
    assert mm.kernel_path(mm.UINT8) == "wgmma_i8"
    _tensor_core_case(torch, mm, "u8", 16384, [("uint8 16384^3", {}, 0)], seed=44, poisons=(0x00, 0xFF))


def test_double_8192_dmma_exact(torch, mm):
    """bench.py double8192: DMMA with the tile height the host picks (0) and forced to 64 rows."""
    assert mm.kernel_path(mm.DOUBLE) == "dmma_f64"
    _tensor_core_case(torch, mm, "dmma", 8192, [("double 8192^3 dmma_tile_rows=0", {"dmma_tile_rows": 0}, 0),
                                                ("double 8192^3 dmma_tile_rows=64", {"dmma_tile_rows": 64}, 0)],
                      seed=45)


def _bench_draw(torch, dtype, n, k, m, lo, hi, seed):
    """bench.py's data: U[lo, hi) drawn in float32, A first, then B, from one seeded generator."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    a = (torch.rand((n, k), generator=g, device="cuda", dtype=torch.float32) * (hi - lo) + lo).to(dtype)
    b = (torch.rand((k, m), generator=g, device="cuda", dtype=torch.float32) * (hi - lo) + lo).to(dtype)
    return a, b


def test_addmin_8192_bit_exact(torch, mm):
    """bench.py addmin8192: float (Add, Min) on U[1, 10) on the ring kernel (default), on semiring_tile_kernel
    (semiring_ring=0) and under MM_FLAG_EXACT, bit for bit against the min-plus reference."""
    n = 8192
    a, b = _bench_draw(torch, torch.float32, n, n, n, 1.0, 10.0, seed=46)
    want = fc.min_plus_reference(torch, a, b)
    settings = [("(Add, Min) float 8192^3 ring", {}, 0),
                ("(Add, Min) float 8192^3 semiring_ring=0", {"semiring_ring": 0}, 0),
                ("(Add, Min) float 8192^3 MM_FLAG_EXACT", {}, mm.FLAG_EXACT)]
    locate_for = lambda knobs: fc.grid_locator("semiring_ring_kernel" if knobs.get("semiring_ring", 1)
                                               else "semiring_tile_kernel", fc.SEMIRING_TILE, fc.SEMIRING_TILE, n, n)
    _run_settings(torch, mm, settings, a, b, want, locate_for, mm.FLOAT, mm.ADD, mm.MIN, "bits")


def test_half_8192_exact_flag_packed_bit_exact(torch, mm):
    """bench.py half8192 --flags 2: the packed HMUL2 / HADD2 path of semiring_tile_kernel on U[0, 1), bit for bit
    against the sequential half reference."""
    n = 8192
    assert mm.kernel_path(mm.HALF, mm.MULTIPLY, mm.ADD, mm.FLAG_EXACT) == "semiring_simt"
    a, b = _bench_draw(torch, torch.float16, n, n, n, 0.0, 1.0, seed=47)
    want = fc.sequential_half_reference(torch, a, b)
    assert bool(torch.isfinite(want).all())
    locate_for = lambda knobs: fc.grid_locator("semiring_tile_kernel", fc.SEMIRING_TILE, fc.SEMIRING_TILE, n, n)
    _run_settings(torch, mm, [("half 8192^3 MM_FLAG_EXACT", {}, mm.FLAG_EXACT)], a, b, want, locate_for, mm.HALF,
                  mm.MULTIPLY, mm.ADD, "bits")


# ---- host-pointer entries ---------------------------------------------------------------------------------------

def _host_case(torch, n, seed):
    a, b = fc.exact_operands(torch, "tf32h", n, n, n, seed, "cuda")
    want = fc.fp64_reference(torch, "tf32h", a, b)
    return a.cpu().numpy(), b.cpu().numpy(), want


def _host_c(n, m, poison=0xFF):
    raw = np.full(n * m * 4 + fc.GUARD, poison, dtype=np.uint8)
    return raw[:n * m * 4].view(np.float32).reshape(n, m), raw[n * m * 4:]


def _check_host(torch, what, c_np, guard_np, want, locate):
    fc.check_guard(torch, what, torch.from_numpy(guard_np), 0xFF)
    fc.compare(torch, what, torch.from_numpy(c_np).cuda(), want, locate, "value", 0xFF)


def test_gemm_host_float_16384_exact(torch, mm):
    """The e2e call of bench.py: Context.gemm_host on host float 16384^3 with the default row chunking, into a
    poisoned host C."""
    n = 16384
    a_np, b_np, want = _host_case(torch, n, seed=48)
    c_np, guard = _host_c(n, n)
    with mm.Context(0) as ctx:
        got, _, _ = ctx.gemm_host(mm.FLOAT, mm.MULTIPLY, mm.ADD, a_np, b_np, n, n, n, out=c_np)
    assert got is c_np
    _check_host(torch, "gemm_host float 16384^3", c_np, guard, want, fc.wgmma_locator(n, n, _sms(torch)))


def _device_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_device_count() < 2, reason="needs two GPUs")
def test_multi_gemm_host_float_16384_exact(torch, mm):
    """bench.py's e2e call with --gpus G: Multi.gemm_host over every GPU of the machine, into a poisoned host C."""
    n = 16384
    gpus = torch.cuda.device_count()
    a_np, b_np, want = _host_case(torch, n, seed=49)
    c_np, guard = _host_c(n, n)
    with mm.Multi(gpus) as multi:
        got, _, _ = multi.gemm_host(mm.FLOAT, mm.MULTIPLY, mm.ADD, a_np, b_np, n, n, n, out=c_np)
        parts = [mm.multi_partition(gpus, g, n, n)[:2] for g in range(gpus)]
    assert got is c_np

    def locate(row, col):
        g = next(i for i, (r0, r1) in enumerate(parts) if r0 <= row < r1)
        r0, r1 = parts[g]
        return "GPU %d (rows %d:%d), its %s" % (g, r0, r1, fc.wgmma_locator(r1 - r0, n, _sms(torch))(row - r0, col))
    _check_host(torch, "Multi.gemm_host float 16384^3 on %d GPUs" % gpus, c_np, guard, want, locate)
