"""GPU tests of bfloat16 (MM_DTYPE_BFLOAT16, run with `-m gpu` on an H100).

* Dense (Multiply, Add) runs on bf16 wgmma with FP32 accumulation and one rounding at the end: on same-sign
  data every element is within 1 bfloat16 ulp of an FP64 evaluation of the same bf16 inputs (the FP32
  accumulation error, relative to sum |a*b|, is far below half an ulp of C when nothing cancels); on mixed-sign
  data the error beyond C's own rounding is bounded relative to sum |a*b|.  Every tuning variant computes the
  same bits, and a transposed A changes nothing.
* MM_FLAG_EXACT and every other semiring are bit-identical to the bfloat16 Naive<> of tests/bf16_naive.py
  (NaN payloads aside).
* Batched calls, the host-pointer entry (also cut into row chunks) and mm_multi agree bit for bit with a
  single enqueue.

Device buffers are torch tensors on cuda:0; the library is called through the C-ABI (ctypes)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bf16_naive  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


@pytest.fixture(scope="module")
def ctx(mm):
    c = mm.Context(0)
    yield c
    c.close()


def _cur(torch):
    return torch.cuda.current_stream().cuda_stream


def _same(x, y):
    import torch
    return torch.equal(x.contiguous().view(-1).view(torch.uint8), y.contiguous().view(-1).view(torch.uint8))


def _randn(torch, shape, seed, scale=1.0):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return (torch.randn(shape, dtype=torch.float32, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _uniform(torch, shape, seed, lo, hi):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return (torch.rand(shape, dtype=torch.float32, device="cuda", generator=g) * (hi - lo) + lo).to(torch.bfloat16)


def _gemm(torch, mm, ctx, a, b, n, k, m, flags=0, map_op=None, reduce_op=None):
    c = torch.empty((n, m), dtype=torch.bfloat16, device="cuda")
    ctx.enqueue(mm.BFLOAT16, mm.MULTIPLY if map_op is None else map_op, mm.ADD if reduce_op is None else reduce_op,
                a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, flags=flags, stream=_cur(torch))
    torch.cuda.synchronize()
    return c


def _ulp(torch, x):
    """The bfloat16 ulp at the binade of each element of x (float64)."""
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


def _ulps_from_fp64(torch, c, a, b):
    """|C - A*B| in units of the bfloat16 ulp at the exact result's binade (FP64 evaluation of the bf16 inputs)."""
    ref = a.double() @ b.double()
    return ((c.double() - ref).abs() / _ulp(torch, ref)).max().item(), ref


@pytest.mark.parametrize("shape", [(256, 256, 256), (513, 544, 544), (1, 32, 32), (128, 4096, 256),
                                   (129, 96, 288), (1024, 1024, 1024)])
def test_tensor_path_within_one_ulp_of_fp64(torch, mm, ctx, shape):
    n, k, m = shape
    a, b = _uniform(torch, (n, k), 1, 0.5, 2.0), _uniform(torch, (k, m), 2, 0.5, 2.0)
    c = _gemm(torch, mm, ctx, a, b, n, k, m)
    worst, _ = _ulps_from_fp64(torch, c, a, b)
    assert worst <= 1.0, worst


@pytest.mark.parametrize("shape", [(513, 544, 544), (128, 4096, 256)])
def test_tensor_path_mixed_signs_bounded_by_sum_of_magnitudes(torch, mm, ctx, shape):
    """Where sums cancel, the FP32 accumulation error is relative to sum |a*b|, not to |C|: within one ulp of C
    plus 2^-14 sum |a*b|."""
    n, k, m = shape
    a, b = _randn(torch, (n, k), 1), _randn(torch, (k, m), 2)
    c = _gemm(torch, mm, ctx, a, b, n, k, m).double()
    ref = a.double() @ b.double()
    mag = a.double().abs() @ b.double().abs()
    assert bool(((c - ref).abs() <= _ulp(torch, ref) + 2.0 ** -14 * mag).all())


def test_tensor_path_range_beyond_half(torch, mm, ctx):
    """C far above 65504 (half's largest value): finite, within 1 ulp."""
    n, k, m = 256, 1024, 256
    a, b = _uniform(torch, (n, k), 3, 100.0, 1000.0), _uniform(torch, (k, m), 4, 100.0, 1000.0)
    c = _gemm(torch, mm, ctx, a, b, n, k, m)
    worst, ref = _ulps_from_fp64(torch, c, a, b)
    assert ref.abs().max().item() > 1e3 * 65504
    assert bool(torch.isfinite(c).all())
    assert worst <= 1.0, worst


def test_every_tuning_variant_gives_the_same_bits(torch, mm, ctx):
    n, k, m = 513, 544, 544
    a, b = _randn(torch, (n, k), 5), _randn(torch, (k, m), 6)
    base = _gemm(torch, mm, ctx, a, b, n, k, m)
    tried = 0
    try:
        for cg in (1, 2):
            for bn in (128, 256):
                for stages in (2, 0):
                    for tma_store in (0, 1):
                        ctx.set_tuning(cta_group=cg, block_n=bn, stages=stages, tma_store=tma_store)
                        assert _same(_gemm(torch, mm, ctx, a, b, n, k, m), base), (cg, bn, stages, tma_store)
                        tried += 1
        ctx.set_tuning(cta_group=2, block_n=256, stages=0, tma_store=1)
        for knobs in (dict(raster_rows=128), dict(raster_rows=65536), dict(l2_policy=1), dict(l2_policy=2),
                      dict(tile_sync=0), dict(tf32_no_round=1)):
            ctx.set_tuning(**knobs)
            assert _same(_gemm(torch, mm, ctx, a, b, n, k, m), base), knobs
            ctx.set_tuning(raster_rows=2048, l2_policy=0, tile_sync=1, tf32_no_round=0)
            tried += 1
    finally:
        ctx.set_tuning(cta_group=2, block_n=256, stages=0, tma_store=1, raster_rows=2048, l2_policy=0, tile_sync=1,
                       tf32_no_round=0)
    assert tried == 22
    # MM_FLAG_TF32X3 does not apply to bf16
    assert _same(_gemm(torch, mm, ctx, a, b, n, k, m, flags=mm.FLAG_TF32X3), base)


def test_transposed_a_gives_the_same_bits(torch, mm, ctx):
    for n, k, m in ((513, 544, 544), (129, 96, 288), (1, 32, 32)):
        a, b = _randn(torch, (n, k), 7), _randn(torch, (k, m), 8)
        row_major = _gemm(torch, mm, ctx, a, b, n, k, m)
        at = a.t().contiguous()   # K x N
        assert _same(_gemm(torch, mm, ctx, at, b, n, k, m, flags=mm.FLAG_TRANSPOSED_A), row_major), (n, k, m)


# ---- exact and semiring paths against the bfloat16 Naive<> ------------------------------------------------------

SPECIAL = np.array([0x7FC0, 0x0000, 0x8000, 0x7F80, 0xFF80, 0x0001, 0x8003, 0x007F, 0x0080, 0x7F7F,
                    0x3F80, 0xBF80, 0x4040, 0xC0A0, 0x3E00, 0x0100, 0x8100], dtype=np.uint16)


def _signed_bits(rng, size, scale=2.0):
    x = (rng.standard_normal(size) * scale).astype(np.float32).view(np.uint32)
    return ((x + 0x7FFF + ((x >> 16) & 1)) >> 16).astype(np.uint16)


_same_nan_free = bf16_naive.same_nan_free


def _datasets(oracle, seed):
    rng = np.random.default_rng(seed)
    a, b = bf16_naive.fill(oracle, 129, 64, 96)
    return [("recipe", a, b, 129, 64, 96, False),
            ("signed_ragged", _signed_bits(rng, 131 * 96), _signed_bits(rng, 96 * 160), 131, 96, 160, False),
            ("special", rng.choice(SPECIAL, 67 * 64), rng.choice(SPECIAL, 64 * 64), 67, 64, 64, False),
            ("transposed", _signed_bits(rng, 64 * 45), _signed_bits(rng, 64 * 96), 45, 64, 96, True)]


@pytest.mark.parametrize("mp", range(5))
def test_semirings_bit_exact_against_naive(mm, ctx, oracle, mp):
    for rd in range(5):
        flags = mm.FLAG_EXACT if (mp, rd) == (mm.MULTIPLY, mm.ADD) else 0
        for name, a, b, n, k, m, ta in _datasets(oracle, 10 * mp + rd):
            f = flags | (mm.FLAG_TRANSPOSED_A if ta else 0)
            got, _, _ = ctx.gemm_host(mm.BFLOAT16, mp, rd, a, b, n, k, m, flags=f)
            want = bf16_naive.naive(mp, rd, a, b, n, k, m, transposed_a=ta)
            assert got.dtype == np.uint16
            assert _same_nan_free(got, want), (mp, rd, name)


def test_packed_paths_with_tuning_ring_off(mm, ctx, oracle):
    """The semiring_ring knob is for 4-byte types; bf16 computes the same bits either way."""
    a, b = bf16_naive.fill(oracle, 129, 64, 96)
    want = bf16_naive.naive(mm.MULTIPLY, mm.ADD, a, b, 129, 64, 96)
    try:
        ctx.set_tuning(semiring_ring=0)
        got, _, _ = ctx.gemm_host(mm.BFLOAT16, mm.MULTIPLY, mm.ADD, a, b, 129, 64, 96, flags=mm.FLAG_EXACT)
    finally:
        ctx.set_tuning(semiring_ring=1)
    assert _same_nan_free(got, want)


def test_ml_dtypes_arrays_round_trip(mm, ctx, oracle):
    ml_dtypes = pytest.importorskip("ml_dtypes")
    a, b = bf16_naive.fill(oracle, 64, 64, 64)
    got, _, _ = ctx.gemm_host(mm.BFLOAT16, mm.ADD, mm.MIN, a.view(ml_dtypes.bfloat16), b.view(ml_dtypes.bfloat16),
                              64, 64, 64)
    assert got.dtype == np.dtype(ml_dtypes.bfloat16)
    assert _same_nan_free(got.view(np.uint16), bf16_naive.naive(mm.ADD, mm.MIN, a, b, 64, 64, 64))


# ---- batched ---------------------------------------------------------------------------------------

BATCH_CONFIGS = [("dense", "MULTIPLY", "ADD", 0), ("exact", "MULTIPLY", "ADD", "EXACT"),
                 ("add_min", "ADD", "MIN", 0), ("transposed", "MULTIPLY", "ADD", "TRANSPOSED_A")]


@pytest.mark.parametrize("cfg", BATCH_CONFIGS, ids=[c[0] for c in BATCH_CONFIGS])
@pytest.mark.parametrize("shape", [(513, 544, 544), (129, 64, 288), (1, 32, 32)])
def test_batched_equals_single_calls(torch, mm, ctx, cfg, shape):
    _, mp, rd, fl = cfg
    mp, rd = getattr(mm, mp), getattr(mm, rd)
    flags = 0 if fl == 0 else getattr(mm, "FLAG_" + fl)
    n, k, m = shape
    for batch in (1, 3, 7):
        for shared_a, shared_b in ((False, False), (True, False), (False, True), (True, True)):
            a = _randn(torch, (1 if shared_a else batch, n * k), batch)
            b = _randn(torch, (1 if shared_b else batch, k * m), batch + 100)
            guard = 4096
            c_raw = torch.full((batch * n * m * 2 + guard,), SENTINEL, dtype=torch.uint8, device="cuda")
            c = c_raw[: batch * n * m * 2].view(torch.bfloat16).view(batch, n * m)
            f = flags | (mm.FLAG_BATCH_SHARED_A if shared_a else 0) | (mm.FLAG_BATCH_SHARED_B if shared_b else 0)
            ctx.enqueue_batched(mm.BFLOAT16, mp, rd, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, batch,
                                flags=f, stream=_cur(torch))
            torch.cuda.synchronize()
            for i in range(batch):
                single = torch.zeros((n * m,), dtype=torch.bfloat16, device="cuda")
                ctx.enqueue(mm.BFLOAT16, mp, rd, a[0 if shared_a else i].data_ptr(), b[0 if shared_b else i].data_ptr(),
                            single.data_ptr(), n, k, m, flags=flags, stream=_cur(torch))
                torch.cuda.synchronize()
                assert _same(single, c[i]), (batch, shared_a, shared_b, i)
            assert bool((c_raw[batch * n * m * 2:] == SENTINEL).all()), (batch, shared_a, shared_b)


def _kernels_launched(torch, fn):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    return [x for x in names if not x.startswith(("Memset", "Memcpy", "[memory]"))]


@pytest.mark.parametrize("mp,rd,fl", [("MULTIPLY", "ADD", 0), ("MULTIPLY", "ADD", "TRANSPOSED_A"),
                                      ("MULTIPLY", "ADD", "EXACT"), ("ADD", "MIN", 0)])
def test_batched_launch_count_equals_single(torch, mm, ctx, mp, rd, fl):
    m_, r_ = getattr(mm, mp), getattr(mm, rd)
    flags = 0 if fl == 0 else getattr(mm, "FLAG_" + fl)
    n, k, m = 129, 64, 160
    expected = mm.launch_count(mm.BFLOAT16, m_, r_, flags)
    for batch in (1, 16):
        a, b = _randn(torch, (batch, n * k), 1), _randn(torch, (batch, k * m), 2)
        c = torch.empty((batch, n * m), dtype=torch.bfloat16, device="cuda")

        def call():
            ctx.enqueue_batched(mm.BFLOAT16, m_, r_, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, batch,
                                flags=flags, stream=_cur(torch))
        call()
        torch.cuda.synchronize()
        kernels = _kernels_launched(torch, call)
        assert len(kernels) == expected, (batch, kernels)


def test_graph_capture_after_reserve_batched(torch, mm, ctx):
    n, k, m, batch = 129, 64, 288, 4
    a, b = _randn(torch, (batch, n * k), 11), _randn(torch, (batch, k * m), 12)
    c = torch.zeros((batch, n * m), dtype=torch.bfloat16, device="cuda")
    ctx.enqueue_batched(mm.BFLOAT16, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, batch,
                        stream=_cur(torch))   # loads the kernels outside any capture
    torch.cuda.synchronize()
    with mm.Context(0) as fresh:
        fresh.reserve_batched(mm.BFLOAT16, n, k, m, batch)
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fresh.enqueue_batched(mm.BFLOAT16, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m,
                                  batch, stream=_cur(torch))
        c.zero_()
        g.replay()
        torch.cuda.synchronize()
        captured = c.clone()
        c.zero_()
        fresh.enqueue_batched(mm.BFLOAT16, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m,
                              batch, stream=_cur(torch))
        torch.cuda.synchronize()
        assert _same(captured, c)
        assert bool(captured.abs().sum() > 0)


# ---- host-pointer entry and mm_multi ---------------------------------------------------------------

def _enqueue_reference(torch, mm, ctx, a_bits, b_bits, n, k, m, mp, rd, flags):
    a = torch.from_numpy(a_bits.astype(np.int16)).cuda().view(torch.bfloat16)
    b = torch.from_numpy(b_bits.astype(np.int16)).cuda().view(torch.bfloat16)
    c = _gemm(torch, mm, ctx, a, b, n, k, m, flags=flags, map_op=mp, reduce_op=rd)
    return c.view(torch.int16).cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("mp,rd,fl", [("MULTIPLY", "ADD", 0), ("MULTIPLY", "ADD", "EXACT"), ("ADD", "MIN", 0)])
def test_host_entry_and_multi_equal_single_enqueue(torch, mm, ctx, mp, rd, fl):
    m_, r_ = getattr(mm, mp), getattr(mm, rd)
    flags = 0 if fl == 0 else getattr(mm, "FLAG_" + fl)
    rng = np.random.default_rng(3)
    n, k, m = 515, 256, 288
    a, b = _signed_bits(rng, n * k), _signed_bits(rng, k * m)
    want = _enqueue_reference(torch, mm, ctx, a, b, n, k, m, m_, r_, flags)
    got, _, _ = ctx.gemm_host(mm.BFLOAT16, m_, r_, a, b, n, k, m, flags=flags)
    assert np.array_equal(got.reshape(-1), want.reshape(-1))
    os.environ["MM_HOST_CHUNK_ROWS"] = "128"        # five row chunks through the H2D / compute / D2H pipeline
    try:
        got, _, _ = ctx.gemm_host(mm.BFLOAT16, m_, r_, a, b, n, k, m, flags=flags)
    finally:
        del os.environ["MM_HOST_CHUNK_ROWS"]
    assert np.array_equal(got.reshape(-1), want.reshape(-1))
    with mm.Multi(2, devices=[0, 0]) as multi:
        got, _, _ = multi.gemm_host(mm.BFLOAT16, m_, r_, a, b, n, k, m, flags=flags)
        assert np.array_equal(got.reshape(-1), want.reshape(-1))
        multi.upload(mm.BFLOAT16, a, b, n, k, m, flags=flags)
        multi.execute(mm.BFLOAT16, m_, r_, n, k, m, flags=flags)
        got = multi.download(mm.BFLOAT16, n, m)
        assert got.dtype == np.uint16 and np.array_equal(got.reshape(-1), want.reshape(-1))
