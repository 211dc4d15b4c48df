"""The tensor-core GEMMs (TF32, 3xTF32, f16, bf16, u8 wgmma and DMMA) against exact or FP64 arithmetic of the same
operation (run with `-m gpu` on an H100).  The restatements are in tests/tensor_numerics.py; the CPU suite
(tests/test_tensor_numerics_cpu.py) shows that each check below rejects plausible wrong kernels.

a. Operand preparation bit for bit through identity products (C = A' I), on every preparation route.
b. Zero-tolerance products on multi-wave schedules: every CTA group runs several tiles, the last wave is partial,
   the rasterisation has a tail group and there are more k-blocks than ring stages; every tuning variant.
c. Batched calls over several waves, each problem against its own exact product.
   Float runs b and c, the edge shapes and the TF32 ties on both of its datapaths: "tf32h" data fits a half and runs
   on the f16 wgmma, "tf32" data carries a row of A times 2^20 and runs on TF32 (tensor_numerics.exact_operands).
   Each call asserts on the host which of the two its operands take.
d. Per-element error bounds on random data (same-sign, mixed-sign, exponent-spread; long K).
e. +-inf, NaN and near-overflow operands: the class of every element as IEEE arithmetic on the prepared operands.

Every C buffer, and 4 KiB after it, is filled with a poison pattern before the call: the guard must be unchanged
and no element of C may still hold the poison.  Bytes 0xFF are NaN in every float type; every byte is a legal
uint8_t result, so uint8_t runs twice, with poison 0x00 and 0xFF.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tensor_numerics as tn  # noqa: E402

pytestmark = pytest.mark.gpu

GUARD = 4096
WGMMA_PATHS = ("tf32", "tf32h", "tf32x3", "f16", "bf16", "u8")

# One shape per family that takes every scheduler path under the default tuning (CG 2, BN 256, raster 2048 rows):
# float: 10 x 18 = 180 tiles on 66 CTA groups (raster groups of 8 + 2 row tiles); with CG 1, BN 128: 19 x 35 = 665
# tiles on 132 CTAs (groups of 16 + 3).  The other families hold the same tile counts at their memory width.
MULTIWAVE = {"tf32": (2305, 272, 4368), "tf32h": (2305, 272, 4368), "tf32x3": (2305, 272, 4368),
             "f16": (2305, 544, 4384), "bf16": (2305, 544, 4384), "u8": (2305, 576, 4416), "dmma": (2305, 264, 4360)}
WIDTH = {"tf32": 16, "tf32h": 16, "tf32x3": 16, "f16": 32, "bf16": 32, "u8": 64, "dmma": 8}

# tuning variants: (knobs, transposed A); raster_rows 768 makes CG 2 groups of 3 + 3 + 3 + 1 row tiles
VARIANTS = ([(dict(cta_group=cg, block_n=bn, tma_store=ts), False) for cg in (1, 2) for bn in (128, 256)
             for ts in (0, 1)]
            + [(dict(stages=2), False), (dict(raster_rows=128), False), (dict(raster_rows=768), False),
               (dict(raster_rows=65536), False), (dict(tile_sync=0), False),
               (dict(), True), (dict(cta_group=1, block_n=128, tma_store=0), True)])


def _vid(v):
    knobs, transposed = v
    return (",".join("%s=%s" % kv for kv in sorted(knobs.items())) or "default") + (",transposed_a" if transposed else "")


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


def _mm_dtype(mm, path):
    return {"tf32": mm.FLOAT, "tf32h": mm.FLOAT, "tf32x3": mm.FLOAT, "f16": mm.HALF, "bf16": mm.BFLOAT16,
            "dmma": mm.DOUBLE, "u8": mm.UINT8}[path]


def _torch_dtype(torch, path):
    return {"tf32": torch.float32, "tf32h": torch.float32, "tf32x3": torch.float32, "f16": torch.float16,
            "bf16": torch.bfloat16, "dmma": torch.float64, "u8": torch.uint8}[path]


def _dev(torch, path, x):
    """A host array of `path`'s input type as a contiguous cuda tensor of the same bytes."""
    x = np.ascontiguousarray(x)
    if path == "bf16":
        return torch.from_numpy(x.view(np.int16)).cuda().view(torch.bfloat16)
    return torch.from_numpy(x).cuda()


def _host(torch, path, c):
    if path == "bf16":
        return c.view(torch.int16).cpu().numpy().view(np.uint16)
    return c.cpu().numpy()


def _gpu_matmul(torch):
    def mul(x, y):
        return torch.matmul(torch.from_numpy(np.ascontiguousarray(x)).cuda(),
                            torch.from_numpy(np.ascontiguousarray(y)).cuda()).cpu().numpy()
    return mul


def _run(torch, mm, ctx, path, a, b, n, k, m, flags=0, batch=None, poison=0xFF):
    """C of one call (batch=None) or one batched call on device operands a, b, into a poisoned buffer; checks the
    guard and that C holds no poison.  Returns C on the host, shaped (batch,) n x m."""
    item = {"tf32": 4, "tf32h": 4, "tf32x3": 4, "f16": 2, "bf16": 2, "dmma": 8, "u8": 1}[path]
    nbytes = (batch or 1) * n * m * item
    raw = torch.full((nbytes + GUARD,), poison, dtype=torch.uint8, device="cuda")
    c = raw[:nbytes].view(_torch_dtype(torch, path))
    f = flags | (mm.FLAG_TF32X3 if path == "tf32x3" else 0)
    stream = torch.cuda.current_stream().cuda_stream
    if batch is None:
        ctx.enqueue(_mm_dtype(mm, path), mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m,
                    flags=f, stream=stream)
    else:
        ctx.enqueue_batched(_mm_dtype(mm, path), mm.MULTIPLY, mm.ADD, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, k, m,
                            batch, flags=f, stream=stream)
    torch.cuda.synchronize()
    assert bool((raw[nbytes:] == poison).all()), "%s: the call wrote past C" % path
    if path != "u8":
        tn.check_no_poison(raw[:nbytes].cpu().numpy(), item, poison)
    out = _host(torch, path, c)
    return out.reshape((batch, n, m) if batch else (n, m))


def _poisons(path):
    return (0x00, 0xFF) if path == "u8" else (0xFF,)


_EXACT_CACHE = {}


def _exact_case(torch, path, n, k, m, seed, batch=1, shared_a=False, shared_b=False, plant="first"):
    """Exact operands (host) and the exact C stored in the output type, from an FP64 product on the GPU (exact for
    integer data).  `plant`: where "tf32" data puts its row times 2^20 (tensor_numerics.plant_rows)."""
    key = (path, n, k, m, seed, batch, shared_a, shared_b, plant)
    if key not in _EXACT_CACHE:
        if len(_EXACT_CACHE) > 4:
            _EXACT_CACHE.clear()
        a, b = tn.exact_operands(path, n, k, m, batch, seed, shared_a, shared_b, plant)
        c64 = torch.matmul(torch.from_numpy(tn.to_float64(path, a)).cuda(),
                           torch.from_numpy(tn.to_float64(path, b)).cuda()).cpu().numpy()
        _EXACT_CACHE[key] = (a, b, tn.store(path, c64))
    return _EXACT_CACHE[key]


# ---- a. preparation through identity products ------------------------------------------------------------------

def _identity_case(path, route, rows=1024, seed=3):
    """(a, b, n, k, m, expected C) with B = I (route a / at) or A = I (route b); the patterns' prepared values
    are C."""
    k = 64
    if path in ("tf32", "tf32x3"):
        # 3xTF32: exponents from 24 up keep lo normal; the two patterns whose hi + lo rounds past FLT_MAX are dropped
        x = tn.tf32_patterns(seed, rows * k, min_exp=24 if path == "tf32x3" else 1)
        if path == "tf32":
            want = tn.rna_tf32(x)
        else:
            hi, lo = tn.split_tf32(x)
            s = hi.astype(np.float64) + lo
            x = np.where(np.abs(s) <= tn.FLT_MAX, x, np.float32(1.5))
            hi, lo = tn.split_tf32(x)
            want = (hi.astype(np.float64) + lo).astype(np.float32)
        eye = np.eye(k, dtype=np.float32)
    else:
        rng = np.random.default_rng(seed)
        if path == "f16":
            bits = rng.integers(0, 1 << 10, rows * k, dtype=np.uint16) | (rng.integers(1, 31, rows * k, dtype=np.uint16) << 10)
            x = (bits | (rng.integers(0, 2, rows * k, dtype=np.uint16) << 15)).view(np.float16)
            eye = np.eye(k, dtype=np.float16)
        elif path == "bf16":
            bits = rng.integers(0, 1 << 7, rows * k, dtype=np.uint16) | (rng.integers(1, 255, rows * k, dtype=np.uint16) << 7)
            x = bits | (rng.integers(0, 2, rows * k, dtype=np.uint16) << 15)
            eye = tn.bf16_naive.from_float(np.eye(k, dtype=np.float32))
        else:
            bits = rng.integers(0, 1 << 52, rows * k, dtype=np.uint64) | (rng.integers(1, 2047, rows * k, dtype=np.uint64) << 52)
            x = (bits | (rng.integers(0, 2, rows * k, dtype=np.uint64) << 63)).view(np.float64)
            eye = np.eye(k, dtype=np.float64)
        want = x
    if route == "b":
        return eye, x.reshape(k, rows), k, k, rows, want.reshape(k, rows)
    return x.reshape(rows, k), eye, rows, k, k, want.reshape(rows, k)


IDENTITY_CASES = [(p, r) for p in ("tf32", "tf32x3") for r in ("a", "at", "b")] + [("f16", "a"), ("bf16", "a"),
                                                                                      ("dmma", "a")]


@pytest.mark.parametrize("path,route", IDENTITY_CASES, ids=["%s-%s" % c for c in IDENTITY_CASES])
def test_identity_product_pins_operand_preparation(torch, mm, ctx, path, route):
    """C = A' I (or I B'): every element is one prepared operand, compared as a number.  TF32: rna_tf32 (ties away
    from zero, the band above 0x7F7FF000 saturating to the largest TF32); 3xTF32: fp32(hi + lo); f16, bf16, double:
    the input."""
    a, b, n, k, m, want = _identity_case(path, route)
    flags = 0
    if route == "at":
        a, flags = np.ascontiguousarray(a.T), mm.FLAG_TRANSPOSED_A
    got = _run(torch, mm, ctx, path, _dev(torch, path, a), _dev(torch, path, b), n, k, m, flags=flags)
    tn.check_exact(path, got, want)


# Subnormal operands: whether the tensor cores keep or flush them (measured on an H100: all kept, pinned here).
SUBNORMALS = {"tf32": "kept", "f16": "kept", "bf16": "kept"}


@pytest.mark.parametrize("path", sorted(SUBNORMALS))
def test_subnormal_operands(torch, mm, ctx, path):
    rng = np.random.default_rng(11)
    rows, k = 256, 64
    if path == "tf32":
        x = (rng.integers(1, 1 << 23, rows * k, dtype=np.uint32) | (rng.integers(0, 2, rows * k, dtype=np.uint32) << 31)).view(np.float32)
        kept, eye = tn.rna_tf32(x), np.eye(k, dtype=np.float32)
    elif path == "f16":
        x = (rng.integers(1, 1 << 10, rows * k, dtype=np.uint16) | (rng.integers(0, 2, rows * k, dtype=np.uint16) << 15)).view(np.float16)
        kept, eye = x, np.eye(k, dtype=np.float16)
    else:
        x = rng.integers(1, 1 << 7, rows * k, dtype=np.uint16) | (rng.integers(0, 2, rows * k, dtype=np.uint16) << 15)
        kept, eye = x, tn.bf16_naive.from_float(np.eye(k, dtype=np.float32))
    got = _run(torch, mm, ctx, path, _dev(torch, path, x.reshape(rows, k)), _dev(torch, path, eye), rows, k, k)
    g, want = tn.to_float64(path, got).reshape(-1), tn.to_float64(path, kept).reshape(-1)
    mode = "kept" if np.array_equal(g, want) else ("flushed" if not np.any(g) else "neither")
    print("subnormal operands on %s: %s" % (path, mode))
    assert mode in ("kept", "flushed")
    if SUBNORMALS[path] is not None:
        assert mode == SUBNORMALS[path]


# ---- b. zero-tolerance products on multi-wave schedules ---------------------------------------------------------

def _assert_datapath(path, a, b):
    """Float: the operands take the datapath that the path key names (a fitting problem runs on the f16 wgmma)."""
    if path in ("tf32", "tf32h"):
        assert tn.datapath(a, b) == path, "%s data that runs on the %s datapath" % (path, tn.datapath(a, b))


def _exact_call(torch, mm, ctx, path, n, k, m, seed, transposed=False, plant="first"):
    a, b, want = _exact_case(torch, path, n, k, m, seed, plant=plant)
    a, b = a[0], b[0]
    _assert_datapath(path, a, b)
    if transposed:
        a = np.ascontiguousarray(a.T)
    da, db = _dev(torch, path, a), _dev(torch, path, b)
    for poison in _poisons(path):
        got = _run(torch, mm, ctx, path, da, db, n, k, m, flags=mm.FLAG_TRANSPOSED_A if transposed else 0,
                   poison=poison)
        tn.check_exact(path, got, want[0])


@pytest.mark.parametrize("variant", VARIANTS, ids=[_vid(v) for v in VARIANTS])
@pytest.mark.parametrize("path", WGMMA_PATHS)
def test_multiwave_exact_every_variant(torch, mm, path, variant):
    knobs, transposed = variant
    n, k, m = MULTIWAVE[path]
    with mm.Context(0) as c:
        c.set_tuning(**knobs)
        _exact_call(torch, mm, c, path, n, k, m, seed=21, transposed=transposed)


@pytest.mark.parametrize("tile_rows", [0, 64, 128])
def test_multiwave_exact_dmma(torch, mm, tile_rows):
    n, k, m = MULTIWAVE["dmma"]
    with mm.Context(0) as c:
        c.set_tuning(dmma_tile_rows=tile_rows)
        _exact_call(torch, mm, c, "dmma", n, k, m, seed=22)


@pytest.mark.parametrize("edge", ["1xWxW", "129x3Wx17W"])
@pytest.mark.parametrize("path", WGMMA_PATHS + ("dmma",))
def test_edge_shapes_exact(torch, mm, ctx, path, edge):
    w = WIDTH[path]
    n, k, m = (1, w, w) if edge == "1xWxW" else (129, 3 * w, 17 * w)
    _exact_call(torch, mm, ctx, path, n, k, m, seed=23, plant="last")
    if path != "dmma":   # DMMA takes a transposed A only for even N
        _exact_call(torch, mm, ctx, path, n, k, m, seed=23, transposed=True, plant="last")


def _tie_call(torch, mm, ctx, route, path):
    """The tie data of `route` on the datapath that `path` names, against the exact product of the rounded operands."""
    n, k, m = 129, 64, 272
    a, b = tn.tie_operands("b" if route == "b" else "a", n, k, m, seed=24)
    if path == "tf32":
        a[n - 1] *= np.float32(tn.PLANT_SCALE)
    _assert_datapath(path, a, b)
    want = tn.store("tf32", tn.rna_tf32(a).astype(np.float64) @ tn.rna_tf32(b).astype(np.float64))
    flags = 0
    if route == "at":
        a, flags = np.ascontiguousarray(a.T), mm.FLAG_TRANSPOSED_A
    got = _run(torch, mm, ctx, "tf32", _dev(torch, "tf32", a), _dev(torch, "tf32", b), n, k, m, flags=flags)
    tn.check_exact("tf32", got, want)


@pytest.mark.parametrize("route", ["a", "at", "b"])
def test_tf32_ties_round_away_from_zero(torch, mm, ctx, route):
    """Odd 12-bit integers are TF32 ties: the exact product of rna-rounded operands pins the rounding mode on the
    row-major A, transposed A and B routes.  The rounded ties are halves, so the call runs on the f16 datapath."""
    _tie_call(torch, mm, ctx, route, "tf32h")


@pytest.mark.parametrize("route", ["a", "at", "b"])
def test_tf32_ties_round_away_from_zero_on_the_tf32_datapath(torch, mm, ctx, route):
    """The same ties with A's last row times 2^20 (still exact): no half holds it, so the call runs on TF32."""
    _tie_call(torch, mm, ctx, route, "tf32")


# ---- c. batched, multi-wave, exact ----------------------------------------------------------------------------

BATCHED = {"tf32": (513, 272, 1040), "tf32h": (513, 272, 1040), "f16": (513, 288, 1088), "u8": (513, 320, 1088),
           "dmma": (513, 272, 1040)}


@pytest.mark.parametrize("shared", ["none", "a", "b"])
@pytest.mark.parametrize("path", sorted(BATCHED))
def test_batched_multiwave_exact(torch, mm, ctx, path, shared):
    """Batch 9: 15 tiles per problem, 135 on 66 CTA groups (the DMMA kernel is not persistent: per-problem offsets).
    Each problem carries its own power-of-two scale and is compared with its own exact product.  "tf32": every copy
    of A has its row times 2^20, first and last rows alternating, the last problem's at its last row."""
    n, k, m = BATCHED[path]
    batch = 9
    sa, sb = shared == "a", shared == "b"
    a, b, want = _exact_case(torch, path, n, k, m, 25, batch, sa, sb)
    flags = (mm.FLAG_BATCH_SHARED_A if sa else 0) | (mm.FLAG_BATCH_SHARED_B if sb else 0)
    for i in range(batch):
        _assert_datapath(path, a[0 if sa else i], b[0 if sb else i])
    da, db = _dev(torch, path, a), _dev(torch, path, b)
    for poison in _poisons(path):
        got = _run(torch, mm, ctx, path, da, db, n, k, m, flags=flags, batch=batch, poison=poison)
        for i in range(batch):
            tn.check_exact(path, got[i], want[i])
    assert want.shape[0] == batch and not np.array_equal(want[0], want[1])   # the problems differ


# ---- d. per-element error bounds --------------------------------------------------------------------------------

BOUND_PATHS = ("tf32", "tf32x3", "f16", "bf16", "dmma")


BOUND_SHAPES = ("513x544x544", "128x16384x256", "multiwave")


@pytest.mark.parametrize("shape", BOUND_SHAPES)
@pytest.mark.parametrize("kind", tn.BOUND_KINDS)
@pytest.mark.parametrize("path", BOUND_PATHS)
def test_error_bound(torch, mm, ctx, path, kind, shape):
    n, k, m = MULTIWAVE[path] if shape == "multiwave" else tuple(int(v) for v in shape.split("x"))
    a, b = tn.bound_operands(path, kind, n, k, m, seed=30 + 3 * tn.BOUND_KINDS.index(kind) + BOUND_SHAPES.index(shape))
    r, s = tn.prepared_product(path, a, b, matmul=_gpu_matmul(torch))
    got = _run(torch, mm, ctx, path, _dev(torch, path, a), _dev(torch, path, b), n, k, m)
    worst, alpha = tn.check_bound(path, got, r, s, k)
    print("bound %-6s %-9s %-13s worst |c-r|/bound %.4f  alpha seen %.5f" % (path, kind, shape, worst, alpha))


# ---- e. special values ------------------------------------------------------------------------------------------

SPECIAL_CASES = [("tf32", False), ("tf32", True), ("tf32x3", False), ("tf32x3", True), ("f16", False),
                 ("bf16", False), ("dmma", False)]


@pytest.mark.parametrize("path,transposed", SPECIAL_CASES,
                         ids=["%s%s" % (p, "-transposed_a" if t else "") for p, t in SPECIAL_CASES])
def test_special_values_follow_ieee(torch, mm, ctx, path, transposed):
    """+-inf and NaN give the class IEEE arithmetic gives on the prepared operands; a near-overflow operand against
    2^-10 stays finite; every finite element is within the bound."""
    n = k = m = 64
    a, b = tn.special_operands(path, n, k, m, seed=26)
    ap, bp = tn.prepared_operands(path, a, b)
    ref = tn.ieee_reference(ap, bp)
    s = tn.ieee_reference(np.abs(ap), np.abs(bp))
    a_in = np.ascontiguousarray(a.T) if transposed else a
    got = _run(torch, mm, ctx, path, _dev(torch, path, a_in), _dev(torch, path, b), n, k, m,
               flags=mm.FLAG_TRANSPOSED_A if transposed else 0)
    tn.check_classes(path, got, ref)
    fin = tn.value_class(ref) == 0
    tn.check_bound(path, got[fin], ref[fin], s[fin], k)
