"""The host-pointer and multi-GPU entries on poisoned staging, against exact results (run with `-m gpu` on an H100).

Entries: Context.gemm_host (mm_gemm_host) in one chunk and in forced row chunks, the default entry
matrix_multiplication_kernel, Multi.gemm_host (mm_multi_gemm_host) over G = 2, 3, 4 with and without chunks inside
each GPU, the upload / execute / download lifecycle, and Context.execute / enqueue on caller-owned device buffers.

Every call under test follows a poison call through the same handle (tests/host_poison.py): the staged A, B,
prepared B and C hold NaN, or for integer types a known constant C in two runs with two constants, and the host C
is prefilled with poison bytes.  A skipped chunk, copy, B slice or column tile therefore shows up as a wrong
element instead of the previous call's correct bytes.  The expected C is computed here, never by the library:

* tensor-core paths (TF32, 3xTF32, f16, bf16, u8 wgmma, DMMA): exact data (tests/tensor_numerics.py) whose product
  is exact in any order, stored once in the output type, compared at zero tolerance;
* CUDA-core paths: the oracle's Naive<> bit for bit (tests/bf16_naive.py for bfloat16); integer (Multiply, Add)
  that wraps around: the exact integer product reduced modulo 2^bits.

Shapes are ragged: N = 1000 is not a multiple of 128 nor of the forced chunk sizes, M = 17 memory words ends in a
partial 128-column tile, and the mm_multi cases cut N unevenly, give some GPUs no rows or no slice of B, and end B in
a short slice.
"""
import os
import sys
from collections import namedtuple

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bf16_naive  # noqa: E402
import host_poison as hp  # noqa: E402
import tensor_numerics as tn  # noqa: E402

pytestmark = pytest.mark.gpu

# codes of include/mm_b200.h
HALF, FLOAT, DOUBLE, INT32, UINT32, UINT8, BF16 = range(7)
MUL, ADD, MIN, MAX = range(4)
TA, EXACT, TF32X3 = 1, 2, 4
NP = {HALF: np.float16, FLOAT: np.float32, DOUBLE: np.float64, INT32: np.int32, UINT32: np.uint32,
      UINT8: np.uint8, BF16: np.uint16}
UNSIGNED = {INT32: np.uint32, UINT32: np.uint32, UINT8: np.uint8}
MM_ERR_INVALID = 1
GUARD = 4096

# data: a tensor_numerics path (exact data) or a draw below; expect: "exact" (the exact product stored once),
# "naive" (Naive<> bit for bit) or "mod" (the exact integer product modulo 2^bits)
Family = namedtuple("Family", "name dtype map reduce flags data expect shape")
FAMILIES = [
    Family("tf32", FLOAT, MUL, ADD, 0, "tf32", "exact", (1000, 256, 272)),
    Family("tf32x3", FLOAT, MUL, ADD, TF32X3, "tf32x3", "exact", (1000, 256, 272)),
    Family("f16", HALF, MUL, ADD, 0, "f16", "exact", (1000, 256, 544)),
    Family("bf16", BF16, MUL, ADD, 0, "bf16", "exact", (1000, 256, 544)),
    Family("u8", UINT8, MUL, ADD, 0, "u8", "exact", (1000, 256, 1088)),
    # K past the 32-bit accumulator headroom of the integer tensor cores: the CUDA-core kernel
    Family("u8_long_k", UINT8, MUL, ADD, 0, "ints", "mod", (130, 33088, 192)),
    Family("dmma", DOUBLE, MUL, ADD, 0, "dmma", "exact", (1000, 256, 136)),
    # transposed A with odd N: the DMMA kernel's 16-byte boxes need even N, so the semiring kernel runs
    Family("f64_ta_odd_n", DOUBLE, MUL, ADD, TA, "dmma", "naive", (999, 256, 136)),
    # 4-byte CUDA-core semirings (the TMA-ring kernel by default); float Min / Max are the FMNMX default on data
    # without NaN whose Map results are never +-0
    Family("f32_add_min", FLOAT, ADD, MIN, 0, "positive", "naive", (1000, 256, 272)),
    Family("f32_mul_min", FLOAT, MUL, MIN, 0, "nonzero", "naive", (1000, 256, 272)),
    Family("f32_add_max", FLOAT, ADD, MAX, 0, "positive", "naive", (1000, 256, 272)),
    Family("i32_mul_add", INT32, MUL, ADD, 0, "ints", "mod", (1000, 256, 272)),
    Family("u32_add_max", UINT32, ADD, MAX, 0, "ints", "naive", (1000, 256, 272)),
    # 1-, 2- and 8-byte semirings; packed __half2 / __nv_bfloat162 for (Multiply, Add) under MM_FLAG_EXACT
    Family("u8_add_max", UINT8, ADD, MAX, 0, "ints", "naive", (1000, 256, 1088)),
    Family("f16_add_min", HALF, ADD, MIN, 0, "signed", "naive", (1000, 256, 544)),
    Family("bf16_max_min", BF16, MAX, MIN, 0, "signed", "naive", (600, 128, 544)),
    Family("f16x2_exact", HALF, MUL, ADD, EXACT, "signed", "naive", (1000, 256, 544)),
    Family("bf16x2_exact", BF16, MUL, ADD, EXACT, "signed", "naive", (600, 128, 544)),
    Family("f64_add_max", DOUBLE, ADD, MAX, 0, "signed", "naive", (1000, 256, 136)),
]
FAM = {f.name: f for f in FAMILIES}
NAMES = [f.name for f in FAMILIES]
ROW_MAJOR = [f.name for f in FAMILIES if not f.flags & TA]      # mm_multi takes row-major A only
RING = ["f32_add_min", "f32_mul_min", "f32_add_max", "i32_mul_add", "u32_add_max"]
CUDA_CORE = [f.name for f in FAMILIES if f.data not in tn.PATHS or f.expect != "exact"]
# MM_HOST_CHUNK_ROWS: the default (one chunk at these sizes), 128 rows (N = 1000: 7 x 128 + 104), 1 (rounds up to
# 128) and N (a chunk of at least N rows)
CHUNKS = ["default", "128", "1", "n"]


def _device_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


# ---- data and expected results ----------------------------------------------------------------------------------

def _draw(fam, rng, shape):
    dt = NP[fam.dtype]
    if fam.data == "ints":
        info = np.iinfo(dt)
        return rng.integers(info.min, info.max, size=shape, dtype=dt, endpoint=True)
    if fam.data == "signed":
        x = rng.standard_normal(shape)
    elif fam.data == "positive":
        x = rng.uniform(0.5, 2.0, shape)
    else:   # "nonzero"
        x = rng.uniform(0.5, 2.0, shape) * rng.choice(np.array([-1.0, 1.0]), size=shape)
    return bf16_naive.from_double(x) if fam.dtype == BF16 else x.astype(dt)


_CASES = {}


def _case(oracle, fam, n, k, m, seed=0):
    """(A n x k, B k x m, expected C, compare) of the family at this shape."""
    key = (fam.name, n, k, m, seed)
    if key not in _CASES:
        if fam.data in tn.PATHS:
            a, b = tn.exact_operands(fam.data, n, k, m, seed=seed)
            a, b = a[0], b[0]
        else:
            rng = np.random.default_rng(seed)
            a, b = _draw(fam, rng, (n, k)), _draw(fam, rng, (k, m))
        if fam.expect == "exact" and fam.data == "u8":
            want = np.mod(a.astype(np.float64) @ b.astype(np.float64), 256).astype(np.uint8)   # < 2^53: exact
        elif fam.expect == "exact":
            want = tn.store(fam.data, tn.to_float64(fam.data, a) @ tn.to_float64(fam.data, b))
        elif fam.expect == "mod":
            wide = a.astype(np.int64).astype(np.uint64) @ b.astype(np.int64).astype(np.uint64)   # wraps mod 2^64
            want = wide.astype(UNSIGNED[fam.dtype]).view(NP[fam.dtype])
        elif fam.dtype == BF16:
            want = bf16_naive.naive(fam.map, fam.reduce, a, b, n, k, m)
        else:
            want = oracle.naive(fam.dtype, fam.map, fam.reduce, a, b, n, k, m, threads=8)
        if fam.expect == "exact":
            path = fam.data
            compare = lambda got, w: tn.check_exact(path, got, w)  # noqa: E731
        else:
            bf16 = fam.dtype == BF16
            compare = lambda got, w: hp.assert_same_bits(got, w, bf16)  # noqa: E731
        _CASES[key] = (a, b, want, compare)
    return _CASES[key]


def check_entry(oracle, entry, fam, n, k, m, transposed_a=False, seed=0):
    """The poisoning protocol around `entry(dtype, map, reduce, a, b, n, k, m, flags, out) -> C`."""
    a, b, want, compare = _case(oracle, fam, n, k, m, seed)
    flags = fam.flags | (TA if transposed_a else 0)
    a_in = np.ascontiguousarray(a.T) if flags & TA else a

    def call(x, y, out, poison):
        mp, rd = (MUL, ADD) if poison else (fam.map, fam.reduce)
        return entry(fam.dtype, mp, rd, x, y, n, k, m, flags, out)

    hp.run(call, a_in.reshape(-1), b.reshape(-1), want, NP[fam.dtype], n, k, m, bf16=fam.dtype == BF16,
           compare=compare)


def context_entry(ctx):
    return lambda dt, mp, rd, a, b, n, k, m, fl, out: ctx.gemm_host(dt, mp, rd, a, b, n, k, m, flags=fl, out=out)[0]


def default_entry(mm):
    return lambda dt, mp, rd, a, b, n, k, m, fl, out: mm.matrix_multiplication_kernel(
        a, b, n, k, m, dtype=dt, map_op=mp, reduce_op=rd, flags=fl, out=out)


def multi_entry(multi):
    return lambda dt, mp, rd, a, b, n, k, m, fl, out: multi.gemm_host(dt, mp, rd, a, b, n, k, m, flags=fl, out=out)[0]


def lifecycle_entry(multi):
    def entry(dt, mp, rd, a, b, n, k, m, fl, out):
        multi.upload(dt, a, b, n, k, m, flags=fl)
        multi.execute(dt, mp, rd, n, k, m, flags=fl)
        return multi.download(dt, n, m, out=out)
    return entry


def _chunks(monkeypatch, chunk, n):
    if chunk == "default":
        monkeypatch.delenv("MM_HOST_CHUNK_ROWS", raising=False)
    else:
        monkeypatch.setenv("MM_HOST_CHUNK_ROWS", str(n) if chunk == "n" else chunk)


# ---- fixtures -----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ctx(mm):
    c = mm.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def staged_ctx(mm):
    """A context whose 4-byte semirings take the register-staged kernel instead of the TMA ring."""
    c = mm.Context(0)
    c.set_tuning(semiring_ring=0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def multis(mm):
    made = {}

    def get(devices):
        key = tuple(devices)
        if key not in made:
            made[key] = mm.Multi(len(key), devices=list(key))
        return made[key]

    yield get
    for multi in made.values():
        multi.close()


# ---- mm_gemm_host -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("name", NAMES)
def test_context_gemm_host(mm, oracle, ctx, monkeypatch, name, chunk):
    fam = FAM[name]
    _chunks(monkeypatch, chunk, fam.shape[0])
    check_entry(oracle, context_entry(ctx), fam, *fam.shape)


@pytest.mark.parametrize("chunk", ["default", "128"])
@pytest.mark.parametrize("name", RING)
def test_context_gemm_host_register_staged_semiring(mm, oracle, staged_ctx, monkeypatch, name, chunk):
    fam = FAM[name]
    _chunks(monkeypatch, chunk, fam.shape[0])
    check_entry(oracle, context_entry(staged_ctx), fam, *fam.shape)


@pytest.mark.parametrize("chunk", ["default", "128"])
@pytest.mark.parametrize("name", NAMES)
def test_default_entry(mm, oracle, monkeypatch, name, chunk):
    fam = FAM[name]
    _chunks(monkeypatch, chunk, fam.shape[0])
    check_entry(oracle, default_entry(mm), fam, *fam.shape)


@pytest.mark.parametrize("name", ROW_MAJOR)
def test_transposed_a_on_context_and_default_entry(mm, oracle, ctx, monkeypatch, name):
    """A stored K x N runs as one chunk whatever MM_HOST_CHUNK_ROWS says."""
    fam = FAM[name]
    monkeypatch.setenv("MM_HOST_CHUNK_ROWS", "128")
    check_entry(oracle, context_entry(ctx), fam, *fam.shape, transposed_a=True)
    check_entry(oracle, default_entry(mm), fam, *fam.shape, transposed_a=True)


# ---- mm_multi_gemm_host and the device-resident lifecycle ---------------------------------------------------------

def _multi_k(fam):
    """K for the row-block split: B's slices (ceil(K / G) rounded up to 64 rows) leave a short last slice, and at
    G = 3 (K = 224) or G = 4 (K = 320) one GPU uploads no slice at all."""
    if fam.name == "u8_long_k":
        return fam.shape[1]
    return 320 if fam.dtype == UINT8 else 224


@pytest.mark.parametrize("chunk", ["default", "128"])
@pytest.mark.parametrize("gpus", [2, 3, 4])
@pytest.mark.parametrize("name", ROW_MAJOR)
def test_multi_gemm_host(mm, oracle, multis, monkeypatch, name, gpus, chunk):
    """On device 0 listed G times: slices of B, the gather, slice tables and host barriers are the NVLink code."""
    fam = FAM[name]
    n, _, m = fam.shape
    _chunks(monkeypatch, chunk, n)
    check_entry(oracle, multi_entry(multis([0] * gpus)), fam, n, _multi_k(fam), m)


# (G, N, K): N < G leaves GPUs without rows; K < 64 G gives fewer slices than GPUs, so some upload nothing
EDGES = [(4, 3, 64), (3, 2, 128), (2, 1, 64), (4, 999, 128)]
EDGE_FAMILIES = ["tf32", "tf32x3", "f16", "bf16", "u8", "dmma", "f32_add_min", "i32_mul_add", "u8_add_max",
                 "bf16_max_min", "f64_add_max"]


@pytest.mark.parametrize("edge", EDGES, ids=lambda e: "G%d-N%d-K%d" % e)
@pytest.mark.parametrize("name", EDGE_FAMILIES)
def test_multi_partition_edges(mm, oracle, multis, monkeypatch, name, edge):
    fam = FAM[name]
    gpus, n, k = edge
    monkeypatch.delenv("MM_HOST_CHUNK_ROWS", raising=False)
    check_entry(oracle, multi_entry(multis([0] * gpus)), fam, n, k, fam.shape[2])
    check_entry(oracle, lifecycle_entry(multis([0] * gpus)), fam, n, k, fam.shape[2])


@pytest.mark.parametrize("gpus", [2, 3])
@pytest.mark.parametrize("name", ROW_MAJOR)
def test_multi_lifecycle(mm, oracle, multis, name, gpus):
    fam = FAM[name]
    n, _, m = fam.shape
    check_entry(oracle, lifecycle_entry(multis([0] * gpus)), fam, n, _multi_k(fam), m)


@pytest.mark.skipif(_device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("chunk", ["default", "128"])
@pytest.mark.parametrize("name", ["tf32", "f16", "bf16", "u8", "dmma", "f32_add_min", "i32_mul_add", "u8_add_max"])
def test_multi_on_distinct_devices(mm, oracle, multis, monkeypatch, name, chunk):
    """B's slices cross NVLink: peer loads in the gather."""
    fam = FAM[name]
    n, _, m = fam.shape
    _chunks(monkeypatch, chunk, n)
    devices = list(range(min(_device_count(), 4)))
    check_entry(oracle, multi_entry(multis(devices)), fam, n, _multi_k(fam), m)
    check_entry(oracle, lifecycle_entry(multis(devices)), fam, n, _multi_k(fam), m)


# ---- what the lifecycle may and may not return --------------------------------------------------------------------

LIFE = FAM["tf32"]
LIFE_SHAPE = (300, 224, 272)


def _assert_refused(mm, multi, shape, known, execute=True):
    """execute (unless execute=False) and download both fail with MM_ERR_INVALID.  If either succeeds, the failure
    names which of the `known` products download returned."""
    n, k, m = shape
    ran = got = None
    if execute:
        try:
            multi.execute(LIFE.dtype, MUL, ADD, n, k, m)
            ran = "execute returned MM_OK"
        except mm.MMError as e:
            assert e.code == MM_ERR_INVALID and "no matching mm_multi_upload" in str(e), str(e)
    try:
        got = multi.download(LIFE.dtype, n, m)
    except mm.MMError as e:
        assert e.code == MM_ERR_INVALID, str(e)
        assert "no matching mm_multi_upload" in str(e) or "no mm_multi_execute" in str(e), str(e)
    if ran or got is not None:
        same = [name for name, w in known.items() if got is not None and hp.same_bits(got, w)]
        pytest.fail("%s; download %s" % (ran or ("execute refused" if execute else "no execute"), "refused" if got is None else
                                         "returned MM_OK with C = " + (" = ".join(same) or "none of the products")))


def _upload_execute(multi, a, b, shape, fam=LIFE):
    n, k, m = shape
    multi.upload(fam.dtype, a, b, n, k, m, flags=fam.flags)
    multi.execute(fam.dtype, fam.map, fam.reduce, n, k, m, flags=fam.flags)


@pytest.mark.parametrize("between", ["same_shape", "smaller", "larger"])
def test_multi_gemm_host_after_upload_invalidates_it(mm, oracle, multis, between):
    """upload(A1, B1); gemm_host(A2, B2); execute must not compute A2 B2 (or a mix) and report success."""
    n, k, m = LIFE_SHAPE
    a1, b1, want1, _ = _case(oracle, LIFE, n, k, m, seed=1)
    shape2 = {"same_shape": (n, k, m), "smaller": (n // 2, k // 2, m), "larger": (2 * n, 2 * k, 2 * m)}[between]
    a2, b2, want2, compare = _case(oracle, LIFE, *shape2, seed=2)
    multi = multis([0, 0])
    multi.upload(LIFE.dtype, a1, b1, n, k, m)
    c2, _, _ = multi.gemm_host(LIFE.dtype, MUL, ADD, a2, b2, *shape2)
    compare(c2, want2)
    _assert_refused(mm, multi, LIFE_SHAPE, {"A1 B1": want1, "A2 B2": want2})


def test_gemm_host_on_a_member_context_invalidates_the_upload(mm, oracle, multis):
    n, k, m = LIFE_SHAPE
    a1, b1, want1, compare = _case(oracle, LIFE, n, k, m, seed=1)
    a2, b2, _, _ = _case(oracle, LIFE, n, k, m, seed=2)
    multi = multis([0, 0])
    for g in range(2):
        _upload_execute(multi, a1, b1, LIFE_SHAPE)
        multi.context(g).gemm_host(LIFE.dtype, MUL, ADD, a2[: n // 2], b2, n // 2, k, m)
        _assert_refused(mm, multi, LIFE_SHAPE, {"A1 B1": want1})
    _upload_execute(multi, a1, b1, LIFE_SHAPE)     # a fresh upload is valid again
    compare(multi.download(LIFE.dtype, n, m), want1)


def test_download_needs_an_execute_after_the_upload(mm, oracle, multis):
    n, k, m = LIFE_SHAPE
    a1, b1, want1, compare = _case(oracle, LIFE, n, k, m, seed=1)
    a2, b2, want2, _ = _case(oracle, LIFE, n, k, m, seed=2)
    multi = multis([0, 0])
    _upload_execute(multi, a1, b1, LIFE_SHAPE)
    compare(multi.download(LIFE.dtype, n, m), want1)
    multi.upload(LIFE.dtype, a2, b2, n, k, m)      # C still holds A1 B1
    _assert_refused(mm, multi, LIFE_SHAPE, {"A1 B1": want1, "A2 B2": want2}, execute=False)


def test_failed_upload_leaves_nothing_resident(mm, oracle, multis):
    n, k, m = LIFE_SHAPE
    a1, b1, want1, _ = _case(oracle, LIFE, n, k, m, seed=1)
    multi = multis([0, 0])
    _upload_execute(multi, a1, b1, LIFE_SHAPE)
    with pytest.raises(mm.MMError) as e:
        multi.upload(LIFE.dtype, a1, b1, n, k + 8, m)       # K not a multiple of the memory width
    assert e.value.code == 2
    _assert_refused(mm, multi, LIFE_SHAPE, {"A1 B1": want1})


def test_upload_that_runs_out_of_memory_leaves_nothing_resident(mm, oracle, multis):
    """An upload whose B cannot be allocated (4 TiB) fails with MM_ERR_NOMEM before copying anything; the earlier
    upload's buffers are gone, so execute and download must refuse."""
    if mm.lib().mm_version() < 203:
        pytest.skip("before version 203 the lifecycle kept the record of a failed upload")
    n, k, m = LIFE_SHAPE
    a1, b1, want1, _ = _case(oracle, LIFE, n, k, m, seed=1)
    multi = multis([0, 0])
    _upload_execute(multi, a1, b1, LIFE_SHAPE)
    with pytest.raises(mm.MMError) as e:
        multi.upload(LIFE.dtype, a1, b1, 2, 1 << 20, 1 << 20)
    assert e.value.code == 4, str(e.value)
    _assert_refused(mm, multi, LIFE_SHAPE, {"A1 B1": want1})


@pytest.mark.parametrize("name", ["tf32", "f32_add_min", "u8"])
def test_lifecycle_repeated_execute_and_second_upload(mm, oracle, multis, name):
    """upload, execute, execute, download; then upload new data, execute, download gives the second product."""
    fam = FAM[name]
    n, _, m = fam.shape
    k = _multi_k(fam)
    a1, b1, want1, compare = _case(oracle, fam, n, k, m, seed=1)
    a2, b2, want2, _ = _case(oracle, fam, n, k, m, seed=2)
    multi = multis([0, 0, 0])
    for want, (a, b) in ((want1, (a1, b1)), (want2, (a2, b2))):
        for rnd in hp.rounds(NP[fam.dtype]):
            pa, pb = hp.poison_operands(NP[fam.dtype], n, k, m, rnd)
            lifecycle_entry(multi)(fam.dtype, MUL, ADD, pa, pb, n, k, m, fam.flags, hp.poison_c(NP[fam.dtype], n, m, rnd))
            multi.upload(fam.dtype, a, b, n, k, m, flags=fam.flags)
            multi.execute(fam.dtype, fam.map, fam.reduce, n, k, m, flags=fam.flags)
            multi.execute(fam.dtype, fam.map, fam.reduce, n, k, m, flags=fam.flags)
            compare(multi.download(fam.dtype, n, m, out=hp.poison_c(NP[fam.dtype], n, m, rnd)), want)


# ---- Context.execute / enqueue on caller-owned device buffers -----------------------------------------------------

@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


DEVICE_CASES = [(name, ta) for name in CUDA_CORE for ta in ([False] if FAM[name].flags & TA else [False, True])]


@pytest.mark.parametrize("how", ["execute", "enqueue"])
@pytest.mark.parametrize("name,ta", DEVICE_CASES, ids=lambda v: v if isinstance(v, str) else ("ta" if v else "rm"))
def test_device_entry_into_poisoned_c(torch, mm, oracle, ctx, name, ta, how):
    """The CUDA-core families into a poisoned C with a 4 KiB guard after it (the tensor-core families have this in
    tests/test_tensor_numerics_gpu.py).  Integer types run with two poison bytes."""
    fam = FAM[name]
    n, k, m = fam.shape
    a, b, want, compare = _case(oracle, fam, n, k, m)
    flags = fam.flags | (TA if ta else 0)
    a_in = np.ascontiguousarray(a.T) if flags & TA else a
    da = torch.from_numpy(a_in.reshape(-1).view(np.uint8).copy()).cuda()
    db = torch.from_numpy(b.reshape(-1).view(np.uint8).copy()).cuda()
    nbytes = n * m * np.dtype(NP[fam.dtype]).itemsize
    for poison in ((0xFF,) if hp.is_float(NP[fam.dtype], fam.dtype == BF16) else (0x5A, 0xA5)):
        raw = torch.full((nbytes + GUARD,), poison, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()                   # the context's stream does not wait for torch's
        if how == "execute":
            ctx.execute(fam.dtype, fam.map, fam.reduce, da.data_ptr(), db.data_ptr(), raw.data_ptr(), n, k, m,
                        flags=flags)
        else:
            ctx.enqueue(fam.dtype, fam.map, fam.reduce, da.data_ptr(), db.data_ptr(), raw.data_ptr(), n, k, m,
                        flags=flags, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert bool((raw[nbytes:] == poison).all()), "the call wrote past C"
        compare(raw[:nbytes].cpu().numpy().view(NP[fam.dtype]).reshape(n, m), want)
