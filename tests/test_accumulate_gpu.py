"""mm_kernel_enqueue_accumulate on an H100 (run with `-m gpu`): C_new == R(C_old, P) byte for byte on every kernel
family, where P is what mm_kernel_enqueue_batched writes for the same arguments on the same device and R is
tests/accumulate_naive.py's restatement of the call's reduce (for Add / Multiply any NaN equals any NaN; Min, Max
and And are compared bit for bit, NaN payloads included).

Every case: P from the plain batched call into its own buffer; C_old drawn by accumulate_naive.c_old from P (random
values, NaN, +-0, +-inf, the identities, P itself and -P); C followed by a 4 KiB guard that must stay as it was.

  wgmma      float at flags 0, MM_FLAG_TF32X3 and MM_FLAG_TRANSPOSED_A, half, bfloat16, uint8_t; each under the
             tuning variants below, at the multi-wave shape of the exact tests and at a ragged edge shape
  DMMA       double, tile rows 0 / 64 / 128, row-major and transposed A
  semirings  every (type, Map, Reduce) under MM_FLAG_EXACT, float Min / Max at flags 0 (FMNMX), semiring_ring = 0 for
             the 4-byte types, transposed A, on accumulate_naive.data (the coverage data of tests/semiring_data.py with
             +0, -0 and NaN products planted for the floating Min / Max); uint8_t (Multiply, Add) with K > 33024,
             checked to run the CUDA-core kernel
  batches    three problems per family under each MM_FLAG_BATCH_SHARED_* combination
  also       graph capture (replayed twice: R(R(C_old, P), P)), profiling, argument validation, and float 16384^3 and
             float (Add, Min) 8192^3 compared on the device
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accumulate_naive as an  # noqa: E402
import full_size_check as fsc  # noqa: E402
import semiring_data as sd  # noqa: E402
from semiring_data import ADD, BF16, DOUBLE, FLOAT, HALF, INT32, MAX, MIN, MULTIPLY, UINT32, UINT8  # noqa: E402

pytestmark = pytest.mark.gpu

TA, EXACT, TF32X3, SHARED_A, SHARED_B = 1, 2, 4, 8, 16
SEED = 7
GUARD_BYTE = 0x5A

# the tensor-core routes: (dtype, flags, multi-wave shape N, K, M of the exact tests)
WGMMA = {"tf32": (FLOAT, 0, (2305, 272, 4368)), "tf32x3": (FLOAT, TF32X3, (2305, 272, 4368)),
         "tf32-ta": (FLOAT, TA, (2305, 272, 4368)), "f16": (HALF, 0, (2305, 544, 4384)),
         "bf16": (BF16, 0, (2305, 544, 4384)), "u8": (UINT8, 0, (2305, 576, 4416))}
EDGE = {FLOAT: (129, 48, 80), HALF: (129, 96, 96), BF16: (65, 160, 96), UINT8: (131, 128, 192)}   # N, K, M
VARIANTS = [dict(), dict(cta_group=1), dict(block_n=128), dict(cta_group=1, block_n=128), dict(tma_store=0),
            dict(tma_store=0, cta_group=1, block_n=128), dict(stages=2), dict(block_n=128, stages=8),
            dict(raster_rows=384)]   # 384 rows: groups of one (CG 2) or three (CG 1) row tiles leave a tail group


def _vid(v):
    return ",".join("%s=%s" % kv for kv in sorted(v.items())) or "default"


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


def _random(dtype, shape, rng):
    if dtype == UINT8:
        return rng.integers(0, 256, size=shape, dtype=np.uint8)
    if dtype in (INT32, UINT32):
        return rng.integers(-1000, 1000, size=shape).astype(sd.NP[dtype])
    return an._round(dtype, rng.uniform(-1.0, 1.0, size=shape))


def _dev(torch, arrays):
    return torch.from_numpy(np.concatenate([np.ascontiguousarray(x).reshape(-1) for x in arrays]).view(np.uint8)
                            .copy()).cuda()


def run(torch, ctx, dt, mp, rd, flags, a_list, b_list, n, k, m, batch=1):
    """P by the plain call, then C_old (+) P by the accumulate call into a guarded C; checked per problem.  a_list /
    b_list: the distinct operands as stored (A transposed when flags has TA)."""
    fmnmx = dt == FLOAT and rd in (MIN, MAX) and not flags & EXACT
    es = sd.SIZE[dt]
    da, db = _dev(torch, a_list), _dev(torch, b_list)
    cbytes = batch * n * m * es
    stream = torch.cuda.current_stream().cuda_stream
    p_dev = torch.zeros(cbytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.enqueue_batched(dt, mp, rd, da.data_ptr(), db.data_ptr(), p_dev.data_ptr(), n, k, m, batch, flags=flags,
                        stream=stream)
    torch.cuda.synchronize()
    p = p_dev.cpu().numpy().view(sd.NP[dt]).reshape(batch, n, m)
    c0 = np.stack([an.c_old(dt, rd, p[z], SEED + z) for z in range(batch)])
    craw = torch.full((cbytes + fsc.GUARD,), GUARD_BYTE, dtype=torch.uint8, device="cuda")
    craw[:cbytes] = torch.from_numpy(c0.reshape(-1).view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    ctx.enqueue_accumulate(dt, mp, rd, da.data_ptr(), db.data_ptr(), craw.data_ptr(), n, k, m, batch=batch,
                           flags=flags, stream=stream)
    torch.cuda.synchronize()
    what = "%s flags %d %dx%dx%d batch %d" % (sd.pair_name(dt, mp, rd), flags, n, k, m, batch)
    fsc.check_guard(torch, what, craw[cbytes:], GUARD_BYTE)
    got = craw[:cbytes].cpu().numpy().view(sd.NP[dt]).reshape(batch, n, m)
    for z in range(batch):
        want = an.reduce_once(dt, rd, c0[z], p[z], fmnmx)
        bad = an.first_difference(dt, got[z], want, rd)
        if bad is not None:
            raise AssertionError("%s problem %d: C differs from R(C_old, P) first at %s: got %r, C_old %r, P %r, "
                                 "want %r" % (what, z, bad, got[z][bad], c0[z][bad], p[z][bad], want[bad]))


# ---- wgmma ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", ["multiwave", "edge"])
@pytest.mark.parametrize("variant", VARIANTS, ids=_vid)
@pytest.mark.parametrize("route", list(WGMMA))
def test_wgmma(torch, mm, route, variant, shape):
    dt, flags, mw = WGMMA[route]
    n, k, m = mw if shape == "multiwave" else EDGE[dt]
    rng = np.random.default_rng([1, dt, flags, n])
    a, b = _random(dt, (n, k), rng), _random(dt, (k, m), rng)
    with mm.Context(0) as ctx:
        ctx.set_tuning(**variant)
        run(torch, ctx, dt, MULTIPLY, ADD, flags, [a.T if flags & TA else a], [b], n, k, m)


# ---- DMMA ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ta", [0, TA])
@pytest.mark.parametrize("tile_rows", [0, 64, 128])
def test_dmma(torch, mm, tile_rows, ta):
    n, k, m = 2306, 264, 4360    # the exact tests' multi-wave shape with an even N: transposed A stays on DMMA
    assert mm.kernel_path(DOUBLE, flags=ta) == "dmma_f64"
    rng = np.random.default_rng([2, tile_rows, ta])
    a, b = _random(DOUBLE, (n, k), rng), _random(DOUBLE, (k, m), rng)
    with mm.Context(0) as ctx:
        ctx.set_tuning(dmma_tile_rows=tile_rows)
        run(torch, ctx, DOUBLE, MULTIPLY, ADD, ta, [a.T if ta else a], [b], n, k, m)


# ---- semirings -----------------------------------------------------------------------------------------------------

PAIRS = [(dt, mp, rd) for dt in sd.TYPES for mp in sd.OPS for rd in sd.OPS]
DEFAULT = [(FLOAT, mp, rd, 0) for mp in sd.OPS for rd in (MIN, MAX)]
STAGED = [(dt, mp, rd, EXACT) for dt, mp, rd in PAIRS if dt in (FLOAT, INT32, UINT32)] + DEFAULT


def _ids(cases):
    return ["%s-f%d" % (sd.pair_name(*c[:3]), c[3]) if len(c) > 3 else sd.pair_name(*c) for c in cases]


@pytest.fixture(scope="module")
def ctx(mm):
    c = mm.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def staged_ctx(mm):
    c = mm.Context(0)
    c.set_tuning(semiring_ring=0)
    yield c
    c.close()


def semiring(torch, c, dt, mp, rd, flags):
    n, m, k = sd.gpu_shape(dt)
    a, b = an.data(dt, mp, rd, n, k, m, 5, exact=bool(flags & EXACT))
    run(torch, c, dt, mp, rd, flags, [a.T if flags & TA else a], [b], n, k, m)


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=_ids(PAIRS))
def test_semiring_exact(torch, ctx, dt, mp, rd):
    semiring(torch, ctx, dt, mp, rd, EXACT)


@pytest.mark.parametrize("dt,mp,rd,flags", DEFAULT, ids=_ids(DEFAULT))
def test_semiring_float_default(torch, ctx, dt, mp, rd, flags):
    semiring(torch, ctx, dt, mp, rd, flags)


@pytest.mark.parametrize("dt,mp,rd,flags", STAGED, ids=_ids(STAGED))
def test_semiring_register_staged(torch, staged_ctx, dt, mp, rd, flags):
    semiring(torch, staged_ctx, dt, mp, rd, flags)


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=_ids(PAIRS))
def test_semiring_transposed_a(torch, ctx, dt, mp, rd):
    semiring(torch, ctx, dt, mp, rd, EXACT | TA)


def test_uint8_long_k_takes_the_cuda_core_kernel(torch, mm, ctx):
    """Past K = 33024 the 32-bit integer accumulators of the tensor cores could overflow: uint8_t (Multiply, Add) runs
    on the CUDA-core kernel, and so does its accumulating call (kernel names read with torch.profiler)."""
    n, m, k = 64, 64, 33088
    assert k > 33024
    rng = np.random.default_rng(3)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(torch, ctx, UINT8, MULTIPLY, ADD, 0, [_random(UINT8, (n, k), rng)], [_random(UINT8, (k, m), rng)], n, k, m)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("semiring_accumulate_tile_kernel" in x for x in names), sorted(set(names))
    assert not any("gemm_wgmma" in x for x in names), sorted(set(names))


# ---- batches -------------------------------------------------------------------------------------------------------

FAMILIES = {"wgmma-tf32": (FLOAT, MULTIPLY, ADD, 0, (257, 272, 96)), "wgmma-f16": (HALF, MULTIPLY, ADD, 0, (257, 288, 96)),
            "wgmma-bf16": (BF16, MULTIPLY, ADD, 0, (130, 96, 64)), "wgmma-u8": (UINT8, MULTIPLY, ADD, 0, (130, 128, 128)),
            "dmma": (DOUBLE, MULTIPLY, ADD, 0, (258, 136, 64)), "ring-f32": (FLOAT, ADD, MIN, EXACT, (259, 272, 160)),
            "tile-i32": (INT32, MAX, ADD, EXACT | TA, (259, 272, 160)), "tile-f16": (HALF, MULTIPLY, ADD, EXACT,
                                                                               (259, 288, 320))}


@pytest.mark.parametrize("shared", [0, SHARED_A, SHARED_B, SHARED_A | SHARED_B])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_batch_of_three(torch, ctx, family, shared):
    dt, mp, rd, flags, (n, m, k) = FAMILIES[family]
    rng = np.random.default_rng([4, dt, shared])
    a = [_random(dt, (n, k), rng) for _ in range(1 if shared & SHARED_A else 3)]
    b = [_random(dt, (k, m), rng) for _ in range(1 if shared & SHARED_B else 3)]
    run(torch, ctx, dt, mp, rd, flags | shared, [x.T if flags & TA else x for x in a], b, n, k, m, batch=3)


# ---- graph capture, profiling, validation ----------------------------------------------------------------------------

@pytest.mark.parametrize("dt,flags", [(FLOAT, 0), (HALF, 0), (DOUBLE, 0), (FLOAT, EXACT)])   # wgmma, DMMA, ring
def test_graph_capture_replayed_twice(torch, mm, dt, flags):
    n, m, k, batch = 257, 288, 128, 2
    rng = np.random.default_rng(5)
    a, b = _random(dt, (batch * n, k), rng), _random(dt, (batch * k, m), rng)
    da, db = _dev(torch, [a]), _dev(torch, [b])
    es = sd.SIZE[dt]
    with mm.Context(0) as c:
        p_dev = torch.zeros(batch * n * m * es, dtype=torch.uint8, device="cuda")
        c.enqueue_batched(dt, MULTIPLY, ADD, da.data_ptr(), db.data_ptr(), p_dev.data_ptr(), n, k, m, batch,
                          flags=flags, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        p = p_dev.cpu().numpy().view(sd.NP[dt])
        c0 = an.c_old(dt, ADD, p, SEED)
        cd = torch.from_numpy(c0.view(np.uint8).copy()).cuda()
        c.reserve_batched(dt, n, k, m, batch, flags=flags)
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            c.enqueue_accumulate(dt, MULTIPLY, ADD, da.data_ptr(), db.data_ptr(), cd.data_ptr(), n, k, m, batch=batch,
                                 flags=flags, stream=s.cuda_stream)
        g.replay()
        g.replay()
        torch.cuda.synchronize()
        got = cd.cpu().numpy().view(sd.NP[dt])
        want = an.reduce_once(dt, ADD, an.reduce_once(dt, ADD, c0, p), p)
        assert an.same(dt, got, want), "R(R(C_old, P), P) after two replays"
        del g
        c.set_profiling(True)
        c.enqueue_accumulate(dt, MULTIPLY, ADD, da.data_ptr(), db.data_ptr(), cd.data_ptr(), n, k, m, batch=batch,
                             flags=flags)
        prep, main, calls = c.profile_read()
        assert calls == 1 and main > 0


def test_argument_validation(torch, mm, ctx):
    n, k, m = 128, 64, 128
    a = torch.zeros(n * k, dtype=torch.float32, device="cuda")
    b = torch.zeros(k * m, dtype=torch.float32, device="cuda")
    c = torch.zeros(n * m, dtype=torch.float32, device="cuda")
    p = (a.data_ptr(), b.data_ptr(), c.data_ptr())
    torch.cuda.synchronize()
    ctx.enqueue_accumulate(FLOAT, MULTIPLY, ADD, *p, n, k, m)   # the valid call
    torch.cuda.synchronize()

    def code(*args, overlap=False, **kw):
        with pytest.raises(mm.MMError) as e:
            ctx.enqueue_accumulate(*args, **kw)
        assert not overlap or "overlap" in str(e.value), str(e.value)
        return e.value.code

    assert code(FLOAT, MULTIPLY, ADD, None, b.data_ptr(), c.data_ptr(), n, k, m) == 1
    assert code(FLOAT, MULTIPLY, ADD, a.data_ptr(), b.data_ptr(), None, n, k, m) == 1
    assert code(FLOAT, MULTIPLY, ADD, a.data_ptr() + 4, b.data_ptr(), c.data_ptr(), n, k, m) == 1
    assert code(FLOAT, MULTIPLY, ADD, *p, n, k, m, batch=0) == 1
    assert code(99, MULTIPLY, ADD, *p, n, k, m) == 1
    assert code(FLOAT, MULTIPLY, ADD, *p, n, 24, m) == 2
    assert code(FLOAT, MULTIPLY, ADD, *p, n, k, m, batch=65536) == 5

    # C overlapping A or B by 16 bytes (the least an aligned C can), with the extents that a batch and its shared
    # operands imply; the same buffers one element further apart are accepted
    es = 4
    big = torch.zeros((2 << 20) // es, dtype=torch.float32, device="cuda")
    base = big.data_ptr()
    for batch, flags in ((1, 0), (3, 0), (3, SHARED_A), (3, SHARED_B), (3, SHARED_A | SHARED_B)):
        na = 1 if flags & SHARED_A else batch
        nb = 1 if flags & SHARED_B else batch
        a_bytes, b_bytes, c_bytes = na * n * k * es, nb * k * m * es, batch * n * m * es
        # C right after A (adjacent: accepted), then one element earlier (overlap: rejected)
        pa, pb = base, base + (1 << 20)
        ctx.enqueue_accumulate(FLOAT, MULTIPLY, ADD, pa, pb, pa + a_bytes, n, k, m, batch=batch, flags=flags)
        assert code(FLOAT, MULTIPLY, ADD, pa, pb, pa + a_bytes - 16, n, k, m, batch=batch, flags=flags,
                    overlap=True) == 1
        # C right before A: C's last element adjacent, then overlapping by one element (16 bytes keep the alignment)
        pa2 = base + 4 * n * m * es
        ctx.enqueue_accumulate(FLOAT, MULTIPLY, ADD, pa2, pb, pa2 - c_bytes, n, k, m, batch=batch, flags=flags)
        assert code(FLOAT, MULTIPLY, ADD, pa2, pb, pa2 - c_bytes + 16, n, k, m, batch=batch, flags=flags,
                    overlap=True) == 1
        # C against B: adjacent after B, then overlapping
        ctx.enqueue_accumulate(FLOAT, MULTIPLY, ADD, pa, pb, pb + b_bytes, n, k, m, batch=batch, flags=flags)
        assert code(FLOAT, MULTIPLY, ADD, pa, pb, pb + b_bytes - 16, n, k, m, batch=batch, flags=flags,
                    overlap=True) == 1
        # ... and C overlapping B by its start
        assert code(FLOAT, MULTIPLY, ADD, pa, pb, pb - c_bytes + 16, n, k, m, batch=batch, flags=flags,
                    overlap=True) == 1
    # A and B may overlap each other
    ctx.enqueue_accumulate(FLOAT, MULTIPLY, ADD, base, base, c.data_ptr(), n, k, m)
    torch.cuda.synchronize()


# ---- full size -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["float-16384", "float-add-min-8192"])
def test_full_size(torch, mm, ctx, case):
    """Every element against the plain call plus torch's add / minimum of the same operands on the device (NaN-free,
    zero-free data: torch.minimum and FMNMX agree there)."""
    n = k = m = 16384 if case == "float-16384" else 8192
    mp, rd = (MULTIPLY, ADD) if case == "float-16384" else (ADD, MIN)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(13)
    a = torch.rand((n, k), generator=gen, device="cuda") * 9 + 1
    b = torch.rand((k, m), generator=gen, device="cuda") * 9 + 1
    c_old = torch.rand((n, m), generator=gen, device="cuda") * 2000 + 1
    p = torch.empty((n, m), device="cuda")
    c = c_old.clone()
    s = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    ctx.enqueue(FLOAT, mp, rd, a.data_ptr(), b.data_ptr(), p.data_ptr(), n, k, m, stream=s)
    ctx.enqueue_accumulate(FLOAT, mp, rd, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m, stream=s)
    torch.cuda.synchronize()
    want = c_old + p if rd == ADD else torch.minimum(c_old, p)
    diff = c.view(torch.int32) != want.view(torch.int32)
    if bool(diff.any()):
        i, j = (int(v) for v in diff.nonzero()[0])
        raise AssertionError("%s: %d elements differ; first (%d, %d): got %r, C_old %r, P %r" % (
            case, int(diff.sum()), i, j, c[i, j].item(), c_old[i, j].item(), p[i, j].item()))
