"""GPU tests of the float GEMM's two datapaths (run with `-m gpu` on an H100): a problem whose TF32-rounded A and B
are all zeros or normal halves runs on the f16 wgmma, any other on TF32.  The choice is made per problem of a batch,
and for the whole A of a call however its rows are split (host-pipeline chunks, devices of mm_multi_gemm_host), so the
batched, chunked and multi-GPU calls keep the single call's bits.  Every C also stays within DESIGN.md section 4's TF32
bound against FP64 of the prepared operands, and holds IEEE's infinities and NaN where the operands carry them."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tensor_numerics as tn  # noqa: E402
import test_float_datapaths_gpu as fd  # noqa: E402

pytestmark = pytest.mark.gpu

N, K, M, BATCH = 260, 192, 144, 4


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


def _problems():
    """Problem 0 fits (U[1, 10)); 1 plants 2^-15, 2^16 and a float subnormal in A's last rows; 2 plants +-inf and NaN
    in B; 3 fits with mixed signs and spread exponents."""
    rng = np.random.default_rng(11)
    a = rng.uniform(1, 10, (BATCH, N, K)).astype(np.float32)
    b = rng.uniform(1, 10, (BATCH, K, M)).astype(np.float32)
    a[1, N - 3, 5], a[1, N - 2, 17], a[1, N - 1, 40] = 2.0 ** -15, 2.0 ** 16, 1e-40
    b[2, 7, 3], b[2, 9, 100], b[2, 50, 60] = np.inf, -np.inf, np.nan
    a[3] = (rng.standard_normal((N, K)) * np.exp2(rng.integers(-6, 6, (N, K)))).astype(np.float32)
    b[3] = (rng.standard_normal((K, M)) * np.exp2(rng.integers(-6, 6, (K, M)))).astype(np.float32)
    return a, b


def _same(x, y):
    """Bit for bit, any NaN equal to any NaN."""
    x, y = np.asarray(x, np.float32).reshape(-1), np.asarray(y, np.float32).reshape(-1)
    nx, ny = np.isnan(x), np.isnan(y)
    return bool(np.array_equal(nx, ny) and np.array_equal(x[~nx].view(np.uint32), y[~ny].view(np.uint32)))


def _check_numerics(c, a, b):
    ap, bp = tn.prepared_operands("tf32", a, b)
    ref = tn.ieee_reference(ap, bp)
    tn.check_classes("tf32", c, ref)
    fin = np.isfinite(ref)
    with np.errstate(invalid="ignore"):
        r, s = ap @ bp, np.abs(ap) @ np.abs(bp)
    tn.check_bound("tf32", np.where(fin, c, 0), np.where(fin, r, 0), np.where(fin, s, 0), K)


def _single(torch, mm, ctx, a, b):
    ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    c = torch.empty((a.shape[0], b.shape[1]), device="cuda")
    s = torch.cuda.current_stream()
    ctx.enqueue(mm.FLOAT, mm.MULTIPLY, mm.ADD, ta.data_ptr(), tb.data_ptr(), c.data_ptr(), a.shape[0], a.shape[1],
                b.shape[1], stream=s.cuda_stream)
    s.synchronize()
    return c.cpu().numpy()


@pytest.fixture(scope="module")
def singles(torch, mm):
    a, b = _problems()
    ctx = mm.Context(0)
    out = [_single(torch, mm, ctx, a[i], b[i]) for i in range(BATCH)]
    ctx.close()
    return a, b, out


def test_single_calls_within_tf32_bound(singles):
    a, b, c = singles
    for i in range(BATCH):
        _check_numerics(c[i], a[i], b[i])


@pytest.mark.parametrize("variant", [{}, {"cta_group": 1, "block_n": 128}, {"tma_store": 0}])
@pytest.mark.parametrize("accumulate", [False, True])
def test_mixed_batch_equals_single_calls(torch, mm, singles, variant, accumulate):
    """One batched call over problems that fit and problems that do not: each C is its single call's (accumulate:
    C_old + that, one float add)."""
    a, b, want = singles
    ctx = mm.Context(0)
    ctx.set_tuning(**variant)
    if variant:
        want = [_single(torch, mm, ctx, a[i], b[i]) for i in range(BATCH)]
    ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    old = torch.from_numpy(np.random.default_rng(2).uniform(-4, 4, (BATCH, N, M)).astype(np.float32)).cuda()
    c = old.clone()
    s = torch.cuda.current_stream()
    call = ctx.enqueue_accumulate if accumulate else ctx.enqueue_batched
    call(mm.FLOAT, mm.MULTIPLY, mm.ADD, ta.data_ptr(), tb.data_ptr(), c.data_ptr(), N, K, M, BATCH, stream=s.cuda_stream)
    s.synchronize()
    ctx.close()
    got, old = c.cpu().numpy(), old.cpu().numpy()
    for i in range(BATCH):
        expect = (old[i] + want[i]).astype(np.float32) if accumulate else want[i]
        assert _same(got[i], expect), (variant, accumulate, i)


@pytest.mark.parametrize("i", range(BATCH))
def test_host_chunks_take_the_whole_a_datapath(mm, singles, monkeypatch, i):
    """mm_gemm_host in 128-row chunks: the planted values sit in the last chunk only."""
    a, b, want = singles
    monkeypatch.setenv("MM_HOST_CHUNK_ROWS", "128")
    with mm.Context(0) as ctx:
        c = ctx.gemm_host(mm.FLOAT, mm.MULTIPLY, mm.ADD, a[i], b[i], N, K, M)[0]
    assert _same(c, want[i]), i


@pytest.mark.parametrize("gpus", [2, 3])
@pytest.mark.parametrize("i", range(BATCH))
def test_multi_gemm_host_takes_the_whole_a_datapath(mm, singles, gpus, i):
    """mm_multi_gemm_host over one device listed several times: the planted values sit in the last device's rows."""
    a, b, want = singles
    with mm.Multi(gpus, devices=[0] * gpus) as multi:
        for rep in range(2):
            c = multi.gemm_host(mm.FLOAT, mm.MULTIPLY, mm.ADD, a[i], b[i], N, K, M)[0]
            assert _same(c, want[i]), (gpus, i, rep)


@pytest.mark.parametrize("gpus", [2, 3])
@pytest.mark.parametrize("i", range(BATCH))
def test_multi_execute_takes_the_whole_a_datapath(mm, singles, gpus, i):
    """mm_multi_upload / execute / download over one device listed several times: each device's rows run as one call
    there, and still take the datapath of the whole A."""
    a, b, want = singles
    with mm.Multi(gpus, devices=[0] * gpus) as multi:
        multi.upload(mm.FLOAT, a[i], b[i], N, K, M)
        for rep in range(2):
            sec_dev, sec_wall = multi.execute(mm.FLOAT, mm.MULTIPLY, mm.ADD, N, K, M)
            assert 0 < sec_dev <= sec_wall
            assert _same(multi.download(mm.FLOAT, N, M), want[i]), (gpus, i, rep)


def test_fitting_problems_run_on_the_f16_datapath(torch, mm):
    """On operands that are exactly halves the rounding is the identity, so tf32_no_round = 1 multiplies the same
    values on the TF32 datapath.  Same-sign data: the f16 datapath rounds its partial sums differently from TF32
    (DESIGN.md §3.1), so a fitting problem gives other bits than TF32, and the same problem with one value of 2^16
    in A (not a half, but TF32-exact) gives exactly TF32's bits (test_float_datapaths_gpu.check_probe_datapaths)."""
    fd.check_probe_datapaths(torch, mm)
