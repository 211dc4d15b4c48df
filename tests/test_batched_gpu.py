"""GPU tests of the batched entry (run with `-m gpu` on an H100): mm_kernel_enqueue_batched computes
`batch` packed problems in the launches of one single call, and every problem's C is BIT-IDENTICAL to
mm_kernel_enqueue on that problem's A and B (same flags, same tuning), for every kernel family.

Buffers are torch tensors on cuda:0; the library is called through the C-ABI (ctypes)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A   # byte pattern of the guard region after C


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


@pytest.fixture(autouse=True)
def stream(torch):
    """Every test runs on its own torch stream, which every library call below is given: torch's work and
    the library's kernels are then stream-ordered."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        yield s.cuda_stream
    s.synchronize()


@pytest.fixture(scope="module")
def ctx(mm):
    c = mm.Context(0)
    yield c
    c.close()


def _tdtype(torch, mm, dtype):
    return {mm.FLOAT: torch.float32, mm.HALF: torch.float16, mm.DOUBLE: torch.float64,
            mm.UINT8: torch.uint8, mm.INT32: torch.int32, mm.UINT32: torch.int32}[dtype]


def _legal(mm, dtype, n, k, m):
    w = mm.memory_width(dtype)
    return n, (k + w - 1) // w * w, (m + w - 1) // w * w


def _random(torch, mm, dtype, shape, gen):
    td = _tdtype(torch, mm, dtype)
    if dtype == mm.UINT8:
        return torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)
    if dtype == mm.INT32:
        return torch.randint(-1000, 1000, shape, dtype=torch.int32, device="cuda", generator=gen)
    # mixed signs: the tensor-core paths must agree bit for bit, not only to a tolerance
    x = torch.randn(shape, dtype=torch.float64, device="cuda", generator=gen)
    return (x * (0.25 if dtype == mm.HALF else 4.0)).to(td)


def _cur(torch):
    return torch.cuda.current_stream().cuda_stream


def _same(x, y):
    import torch
    return torch.equal(x.contiguous().view(-1).view(torch.uint8), y.contiguous().view(-1).view(torch.uint8))


def run_batched_vs_single(torch, mm, ctx, dtype, mp, rd, flags, n, k, m, batch, shared_a, shared_b, seed=1,
                          poison=None):
    """Runs one batched enqueue and `batch` single enqueues; returns (list of problems whose C differs,
    guard region untouched).  `poison(a, b)` may modify the packed operands before the runs."""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    na, nb = (1 if shared_a else batch), (1 if shared_b else batch)
    a = _random(torch, mm, dtype, (na, n * k), gen)
    b = _random(torch, mm, dtype, (nb, k * m), gen)
    if poison is not None:
        poison(a, b)
    guard = 4096
    td = _tdtype(torch, mm, dtype)
    es = torch.tensor([], dtype=td).element_size()
    c_raw = torch.full((batch * n * m * es + guard,), SENTINEL, dtype=torch.uint8, device="cuda")
    c = c_raw[: batch * n * m * es].view(td).view(batch, n * m)
    single = torch.empty((n * m,), dtype=td, device="cuda")
    f = flags | (mm.FLAG_BATCH_SHARED_A if shared_a else 0) | (mm.FLAG_BATCH_SHARED_B if shared_b else 0)
    stream = _cur(torch)
    ctx.enqueue_batched(dtype, mp, rd, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, batch, flags=f, stream=stream)
    torch.cuda.synchronize()
    bad = []
    for i in range(batch):
        ai, bi = a[0 if shared_a else i], b[0 if shared_b else i]
        single.fill_(0)
        ctx.enqueue(dtype, mp, rd, ai.data_ptr(), bi.data_ptr(), single.data_ptr(), n, k, m, flags=flags, stream=stream)
        torch.cuda.synchronize()
        if not _same(single, c[i]):
            bad.append(i)
    guard_ok = bool((c_raw[batch * n * m * es:] == SENTINEL).all())
    return bad, guard_ok


# (name, dtype, map, reduce, flags, tuning)
CONFIGS = [
    ("wgmma_tf32", "FLOAT", "MULTIPLY", "ADD", 0, {}),
    ("wgmma_f16", "HALF", "MULTIPLY", "ADD", 0, {}),
    ("wgmma_i8", "UINT8", "MULTIPLY", "ADD", 0, {}),
    ("dmma_f64", "DOUBLE", "MULTIPLY", "ADD", 0, {}),
    ("semiring_ring", "FLOAT", "ADD", "MIN", 0, {}),
    ("semiring_staged", "FLOAT", "ADD", "MIN", 0, {"semiring_ring": 0}),
    ("exact", "FLOAT", "MULTIPLY", "ADD", "EXACT", {}),
    ("tf32x3", "FLOAT", "MULTIPLY", "ADD", "TF32X3", {}),
    ("transposed_tf32", "FLOAT", "MULTIPLY", "ADD", "TRANSPOSED_A", {}),
    ("transposed_i8", "UINT8", "MULTIPLY", "ADD", "TRANSPOSED_A", {}),
    ("transposed_f64", "DOUBLE", "MULTIPLY", "ADD", "TRANSPOSED_A", {}),
    ("transposed_semiring", "INT32", "ADD", "MIN", "TRANSPOSED_A", {}),
]
SHAPES = [(513, 528, 528), (129, 48, 272), (1, 16, 16)]
SHAPE_F64 = (130, 40, 136)   # double: K = 40 ends inside a BK = 32 k-tile
SHARES = [(False, False), (True, False), (False, True), (True, True)]
CASES = [(cfg, shape) for cfg in CONFIGS for shape in SHAPES + ([SHAPE_F64] if cfg[1] == "DOUBLE" else [])]


def _resolve(mm, cfg):
    name, dt, mp, rd, fl, tune = cfg
    flags = 0 if fl == 0 else getattr(mm, "FLAG_" + fl)
    return getattr(mm, dt), getattr(mm, mp), getattr(mm, rd), flags, tune


@pytest.mark.parametrize("shared", SHARES, ids=["packed", "shared_a", "shared_b", "shared_ab"])
@pytest.mark.parametrize("cfg,shape", CASES, ids=["%s-%dx%dx%d" % ((c[0],) + s) for c, s in CASES])
def test_batched_equals_single_calls(torch, mm, ctx, cfg, shape, shared):
    """Shapes are scaled per type to its memory width (K and M rounded up)."""
    dtype, mp, rd, flags, tune = _resolve(mm, cfg)
    n, k, m = _legal(mm, dtype, *shape)
    ctx.set_tuning(**tune)
    try:
        for batch in (1, 3, 7):
            bad, guard_ok = run_batched_vs_single(torch, mm, ctx, dtype, mp, rd, flags, n, k, m, batch, *shared,
                                                  seed=batch)
            assert not bad, "batch %d: problems %s differ from their single calls" % (batch, bad)
            assert guard_ok, "batch %d wrote past the end of C" % batch
    finally:
        ctx.set_tuning(semiring_ring=1)


@pytest.mark.parametrize("dt", ["FLOAT", "HALF", "UINT8"])
def test_batched_identical_across_tuning_variants(torch, mm, ctx, dt):
    dtype = getattr(mm, dt)
    results = []
    for shape, shared_b in (((513, 528, 528), False), ((129, 48, 272), True)):
        n, k, m = _legal(mm, dtype, *shape)
        gen = torch.Generator(device="cuda")
        gen.manual_seed(7)
        a = _random(torch, mm, dtype, (3, n * k), gen)
        b = _random(torch, mm, dtype, (1 if shared_b else 3, k * m), gen)
        outs = []
        try:
            for cg in (1, 2):
                for bn in (128, 256):
                    for tma_store in (0, 1):
                        ctx.set_tuning(cta_group=cg, block_n=bn, tma_store=tma_store)
                        c = torch.zeros((3, n * m), dtype=_tdtype(torch, mm, dtype), device="cuda")
                        ctx.enqueue_batched(dtype, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(),
                                            n, k, m, 3, flags=mm.FLAG_BATCH_SHARED_B if shared_b else 0,
                                            stream=_cur(torch))
                        s = torch.zeros((n * m,), dtype=c.dtype, device="cuda")
                        ctx.enqueue(dtype, mm.MULTIPLY, mm.ADD, a[2].data_ptr(), b[0 if shared_b else 2].data_ptr(),
                                    s.data_ptr(), n, k, m, stream=_cur(torch))
                        torch.cuda.synchronize()
                        assert _same(s, c[2]), (cg, bn, tma_store)
                        outs.append(c)
        finally:
            ctx.set_tuning(cta_group=2, block_n=256, tma_store=1)
        for o in outs[1:]:
            assert _same(o, outs[0])
        results.append(len(outs))
    assert results == [8, 8]


def _poison(torch, mm, dtype, n, k, m, shared_a, shared_b):
    """NaN / +-Inf (or 0xFF bytes for integers) throughout problem 1's A and B."""
    def apply(a, b):
        for t, shared in ((a, shared_a), (b, shared_b)):
            if shared:
                continue
            x = t[1]
            if dtype in (mm.UINT8, mm.INT32):
                x.fill_(-1 if dtype == mm.INT32 else 255)
            else:
                x[0::3] = float("nan")
                x[1::3] = float("inf")
                x[2::3] = float("-inf")
    return apply


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_no_leakage_between_problems(torch, mm, ctx, cfg):
    """Problem 1 carries NaN / Inf; problems 0 and 2 (ragged in every dimension) must still equal their
    single calls byte for byte, and nothing may be written past the end of C."""
    dtype, mp, rd, flags, tune = _resolve(mm, cfg)
    shape = SHAPE_F64 if dtype == mm.DOUBLE else (129, 48, 272)
    n, k, m = _legal(mm, dtype, *shape)
    ctx.set_tuning(**tune)
    try:
        for shared_a, shared_b in SHARES:
            bad, guard_ok = run_batched_vs_single(torch, mm, ctx, dtype, mp, rd, flags, n, k, m, 3, shared_a, shared_b,
                                                  poison=_poison(torch, mm, dtype, n, k, m, shared_a, shared_b))
            assert not bad, (shared_a, shared_b, bad)
            assert guard_ok
    finally:
        ctx.set_tuning(semiring_ring=1)


@pytest.mark.parametrize("dt,mp,rd,shape", [("FLOAT", "ADD", "MIN", (129, 48, 144)),
                                            ("INT32", "MULTIPLY", "ADD", (65, 64, 96)),
                                            ("UINT8", "MULTIPLY", "ADD", (129, 128, 192))])
def test_batched_against_oracle(torch, mm, ctx, oracle, dt, mp, rd, shape):
    dtype, m_, r_ = getattr(mm, dt), getattr(mm, mp), getattr(mm, rd)
    n, k, m = shape
    batch = 3
    data = [oracle.fill(dtype, n, k, m, 30 + i) for i in range(batch)]
    a = torch.from_numpy(np.stack([x[0].reshape(-1) for x in data])).cuda()
    b = torch.from_numpy(np.stack([x[1].reshape(-1) for x in data])).cuda()
    c = torch.empty((batch, n * m), dtype=a.dtype, device="cuda")
    ctx.enqueue_batched(dtype, m_, r_, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, batch, stream=_cur(torch))
    torch.cuda.synchronize()
    got = c.cpu().numpy()
    for i, (ai, bi) in enumerate(data):
        ref = oracle.naive(dtype, m_, r_, ai, bi, n, k, m, threads=8)
        assert got[i].tobytes() == ref.reshape(-1).tobytes(), "problem %d" % i


def _kernels_launched(torch, fn):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    return [x for x in names if not x.startswith(("Memset", "Memcpy", "[memory]"))]


@pytest.mark.parametrize("dt,mp,rd,fl", [("FLOAT", "MULTIPLY", "ADD", 0), ("FLOAT", "MULTIPLY", "ADD", "TF32X3"),
                                         ("HALF", "MULTIPLY", "ADD", "TRANSPOSED_A"), ("UINT8", "MULTIPLY", "ADD", 0),
                                         ("DOUBLE", "MULTIPLY", "ADD", 0), ("FLOAT", "ADD", "MIN", 0)])
def test_launch_count_independent_of_batch(torch, mm, ctx, dt, mp, rd, fl):
    dtype, m_, r_ = getattr(mm, dt), getattr(mm, mp), getattr(mm, rd)
    flags = 0 if fl == 0 else getattr(mm, "FLAG_" + fl)
    n, k, m = _legal(mm, dtype, 129, 64, 136)
    expected = mm.launch_count(dtype, m_, r_, flags)
    for batch in (1, 16):
        for shared in (0, mm.FLAG_BATCH_SHARED_B):
            gen = torch.Generator(device="cuda")
            a = _random(torch, mm, dtype, (batch, n * k), gen)
            b = _random(torch, mm, dtype, (batch, k * m), gen)
            c = torch.empty((batch, n * m), dtype=a.dtype, device="cuda")

            def call():
                ctx.enqueue_batched(dtype, m_, r_, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, batch,
                                    flags=flags | shared, stream=_cur(torch))
            call()                     # warm-up: scratch, module loading
            torch.cuda.synchronize()
            kernels = _kernels_launched(torch, call)
            assert len(kernels) == expected, (batch, shared, kernels)


def test_profiling_counts_one_call_per_batched_call(torch, mm, ctx):
    n, k, m, batch = 128, 64, 128, 5
    a = torch.ones((batch, n * k), device="cuda")
    b = torch.ones((batch, k * m), device="cuda")
    c = torch.empty((batch, n * m), device="cuda")
    ctx.set_profiling(True)
    try:
        for _ in range(2):
            ctx.enqueue_batched(mm.FLOAT, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(),
                n, k, m, batch, stream=_cur(torch))
        prep, main, calls = ctx.profile_read()
    finally:
        ctx.set_profiling(False)
    assert calls == 2 and prep > 0 and main > 0
    assert float(c[4, 0]) == 64.0


def test_graph_capture_after_reserve_batched(torch, mm, ctx):
    n, k, m, batch = 129, 48, 272, 4
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    a = _random(torch, mm, mm.FLOAT, (batch, n * k), gen)
    b = _random(torch, mm, mm.FLOAT, (batch, k * m), gen)
    c = torch.zeros((batch, n * m), device="cuda")
    # load the kernels outside any capture (another context: the ones below start with no scratch)
    ctx.enqueue_batched(mm.FLOAT, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(),
        n, k, m, batch, stream=_cur(torch))
    torch.cuda.synchronize()
    with mm.Context(0) as fresh:
        s = torch.cuda.Stream()
        # without a reserve, the first call is captured and its scratch would have to grow: refused
        g0 = torch.cuda.CUDAGraph()
        with pytest.raises(mm.MMError) as e:
            with torch.cuda.graph(g0, stream=s):
                fresh.enqueue_batched(mm.FLOAT, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m,
                                    batch, stream=_cur(torch))
        assert e.value.code == 1 and "reserve" in str(e.value)
    torch.cuda.synchronize()
    with mm.Context(0) as fresh:
        fresh.reserve_batched(mm.FLOAT, n, k, m, batch)
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fresh.enqueue_batched(mm.FLOAT, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m,
                                batch, stream=_cur(torch))
        g.replay()
        torch.cuda.synchronize()
        captured = c.clone()
        c.zero_()
        fresh.enqueue_batched(mm.FLOAT, mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(),
            n, k, m, batch, stream=_cur(torch))
        torch.cuda.synchronize()
        assert _same(captured, c)
        c.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert _same(captured, c)


def test_validation(torch, mm, ctx):
    a = torch.zeros((2, 64 * 64), device="cuda")
    p = a.data_ptr()
    enq = mm.lib().mm_kernel_enqueue_batched

    def rc(n, k, m, batch, ptr=p, dtype=mm.FLOAT):
        return enq(ctx._h, dtype, mm.MULTIPLY, mm.ADD, 0, ptr, ptr, ptr, n, k, m, batch, None)
    assert rc(64, 64, 64, 0) == 1                       # MM_ERR_INVALID
    assert rc(64, 64, 64, 65536) == 5                   # MM_ERR_UNSUPPORTED
    assert "65535" in mm.lib().mm_last_error().decode()
    assert rc(1 << 21, 64, 64, 1024) == 5               # batch * N = 2^31
    assert rc(64, 1 << 21, 64, 1024) == 5               # batch * K
    assert rc(64, 64, 1 << 21, 1024) == 5               # batch * M
    assert rc(64, 64, 64, 2, ptr=p + 4) == 1            # misaligned
    assert rc(64, 24, 64, 2) == 2                       # the single call's shape rule
    assert mm.lib().mm_context_reserve_batched(ctx._h, mm.FLOAT, 0, 64, 64, 64, 0) == 1
    assert mm.lib().mm_context_reserve_batched(ctx._h, mm.FLOAT, 0, 64, 64, 64, 70000) == 5
    torch.cuda.synchronize()
