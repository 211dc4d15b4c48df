"""GPU parity at BASELINE.json's FULL sizes, where the oracle cannot run the whole problem: sampled
rows against the oracle plus size-independent properties (checksum of checksums, exact linearity
under power-of-two scaling, row-block consistency).  Device-resident data, C-ABI launches."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _device_problem(torch, dtype, n, k, m, lo=1.0, hi=10.0, seed=5):
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    a = (torch.rand((n, k), generator=gen, device=dev, dtype=torch.float32) * (hi - lo) + lo).to(dtype)
    b = (torch.rand((k, m), generator=gen, device=dev, dtype=torch.float32) * (hi - lo) + lo).to(dtype)
    return a, b, torch.empty((n, m), device=dev, dtype=dtype)


def _launch(mm, ctx, torch, dt, mp, rd, a, b, c, flags=0):
    n, k = a.shape
    m = b.shape[1]
    s = torch.cuda.current_stream()
    # the context's own stream is non-blocking: it does not wait for torch's pending work (the kernels that
    # generate A and B, or an earlier fill of C) unless the device is idle first
    torch.cuda.synchronize()
    ctx.enqueue(dt, mp, rd, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, flags=flags,
                stream=s.cuda_stream if s.cuda_stream else None)
    torch.cuda.synchronize()


def test_float_16384_cubed_properties(mm, oracle):
    """BASELINE config 2: float 16384^3 on the tensor-core path."""
    torch = pytest.importorskip("torch")
    n = k = m = 16384
    a, b, c = _device_problem(torch, torch.float32, n, k, m)
    with mm.Context(0) as ctx:
        _launch(mm, ctx, torch, mm.FLOAT, mm.MULTIPLY, mm.ADD, a, b, c)
        # (1) sampled rows against the oracle's Naive<> (reference criterion 1e-3, suite tolerance 5e-4)
        rows = [0, 8191, 16383]
        b_host = b.cpu().numpy()
        for r in rows:
            ref = oracle.naive(oracle.FLOAT, oracle.MULTIPLY, oracle.ADD, a[r:r + 1].cpu().numpy(), b_host, 1, k, m,
                               threads=8)
            got = c[r:r + 1].cpu().numpy()
            assert oracle.verify(oracle.FLOAT, got, ref) == -1
            assert float(np.max(np.abs(got.astype(np.float64) - ref) / ref)) <= 5e-4
        # (2) checksum of checksums: C.1 == A.(B.1), evaluated in FP64 on the device
        ones = torch.ones((m,), device=a.device, dtype=torch.float64)
        lhs = c.double() @ ones
        rhs = a.double() @ (b.double() @ ones)
        assert float(((lhs - rhs).abs() / rhs).max()) <= 2e-4
        # (3) exact linearity under power-of-two scaling: rounding to TF32 commutes with *2, so
        #     (2A).B must equal 2.(A.B) BIT FOR BIT
        c2 = torch.empty_like(c)
        _launch(mm, ctx, torch, mm.FLOAT, mm.MULTIPLY, mm.ADD, a * 2.0, b, c2)
        assert torch.equal(c2, c * 2.0)
        # (4) row-block consistency (the multi-GPU partition): rows [4096, 6144) computed alone
        cb = torch.empty((2048, m), device=a.device, dtype=torch.float32)
        _launch(mm, ctx, torch, mm.FLOAT, mm.MULTIPLY, mm.ADD, a[4096:6144].contiguous(), b, cb)
        assert torch.equal(cb, c[4096:6144])


def test_addmin_8192_cubed_sampled_rows_bit_exact(mm, oracle):
    """BASELINE config 5: (Add, Min) float 8192^3 — sampled rows bit-exact against the oracle."""
    torch = pytest.importorskip("torch")
    n = k = m = 8192
    a, b, c = _device_problem(torch, torch.float32, n, k, m)
    with mm.Context(0) as ctx:
        _launch(mm, ctx, torch, mm.FLOAT, mm.ADD, mm.MIN, a, b, c)
        b_host = b.cpu().numpy()
        for r in (0, 4097, 8191):
            ref = oracle.naive(oracle.FLOAT, oracle.ADD, oracle.MIN, a[r:r + 1].cpu().numpy(), b_host, 1, k, m, threads=8)
            assert c[r:r + 1].cpu().numpy().tobytes() == ref.tobytes()
        # min-plus is monotone: adding a constant to A shifts C by exactly that constant when it is
        # representable without rounding (power of two, same binade growth is checked by the oracle rows)
        # idempotence of the row-block split
        cb = torch.empty((1024, m), device=a.device, dtype=torch.float32)
        _launch(mm, ctx, torch, mm.FLOAT, mm.ADD, mm.MIN, a[3072:4096].contiguous(), b, cb)
        assert torch.equal(cb, c[3072:4096])


def test_double_8192_cubed_properties(mm, oracle):
    """BASELINE config 4: double 8192^3 on the DMMA path."""
    torch = pytest.importorskip("torch")
    n = k = m = 8192
    a, b, c = _device_problem(torch, torch.float64, n, k, m)
    with mm.Context(0) as ctx:
        _launch(mm, ctx, torch, mm.DOUBLE, mm.MULTIPLY, mm.ADD, a, b, c)
        b_host = b.cpu().numpy()
        for r in (0, 8191):
            ref = oracle.naive(oracle.DOUBLE, oracle.MULTIPLY, oracle.ADD, a[r:r + 1].cpu().numpy(), b_host, 1, k, m,
                               threads=8)
            got = c[r:r + 1].cpu().numpy()
            assert float(np.max(np.abs(got - ref) / ref)) <= 1e-12
        ones = torch.ones((m,), device=a.device, dtype=torch.float64)
        lhs, rhs = c @ ones, a @ (b @ ones)
        assert float(((lhs - rhs).abs() / rhs).max()) <= 1e-11
        c2 = torch.empty_like(c)
        _launch(mm, ctx, torch, mm.DOUBLE, mm.MULTIPLY, mm.ADD, a * 2.0, b, c2)
        assert torch.equal(c2, c * 2.0)


def test_half_32768_cubed_properties(mm, oracle):
    """BASELINE config 3: half 32768^3 (inputs in [0, 1) so that C stays finite in half)."""
    torch = pytest.importorskip("torch")
    n = k = m = 32768
    a, b, c = _device_problem(torch, torch.float16, n, k, m, lo=0.0, hi=1.0)
    with mm.Context(0) as ctx:
        _launch(mm, ctx, torch, mm.HALF, mm.MULTIPLY, mm.ADD, a, b, c)
        assert bool(torch.isfinite(c[::4097]).all())
        # sampled rows against an FP64 evaluation of the same half inputs (tolerance 1e-3: one rounding to half)
        for r in (0, 16384, 32767):
            ref = a[r:r + 1].double() @ b.double()
            rel = ((c[r:r + 1].double() - ref).abs() / ref).max()
            assert float(rel) <= 1e-3
        # exact linearity under power-of-two scaling (no overflow: C < 16384 * 0.5)
        c2 = torch.empty_like(c)
        _launch(mm, ctx, torch, mm.HALF, mm.MULTIPLY, mm.ADD, a * 2.0, b, c2)
        assert torch.equal(c2[::513], (c * 2.0)[::513])
