"""The float GEMM's two datapaths (run with `-m gpu` on an H100).  A float (Multiply, Add) problem whose TF32-rounded A
and B are all zeros or normal halves (tensor_numerics.fits_half) runs on the f16 wgmma, any other on TF32; the
persistent kernel picks the datapath per tile from its problem's fits words, and the two datapaths run different
k-block counts over one shared-memory ring.

* The datapath probe: on same-sign, fp16-exact U[1, 10) data the TF32 rounding is the identity, so
  `tf32_no_round = 1` multiplies the same values on TF32.  A problem that ran on TF32 equals that bit for bit; one
  that ran on f16 differs in most elements, because the f16 datapath rounds its partial sums differently (DESIGN.md
  section 3.1).
1. CTAs that switch datapath: batches whose fitting and non-fitting problems alternate along each CTA group's tile
   sequence (a host restatement of the schedule chooses them), under every tuning variant, at K = 272 (9 TF32 and 5
   f16 k-blocks) and K = 16 (one partial k-block).  Exact data: each problem equals its exact product; probe data:
   each problem equals its own single call and is classified by the probe.
2. The same batches through mm_kernel_enqueue_accumulate, C_old on the exact grid of C, so C_old + P is exact.
3. Values that cross the fits boundary only through rounding, at the last element and at an interior 64 x 64 tile
   edge of every preparation route, against zeros of the other operand.
4. The fits words are per call: alternating calls in one context, and replays of a captured graph whose operand
   contents cross the boundary.

Every C, and 4 KiB after it, is poisoned first (test_tensor_numerics_gpu._run).
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_size_check as fc  # noqa: E402
import tensor_numerics as tn  # noqa: E402
import test_tensor_numerics_gpu as tng  # noqa: E402

pytestmark = pytest.mark.gpu

VARIANTS = tng.VARIANTS
SWITCH_N, SWITCH_M = 320, 272          # 2 x 2 tiles of 256 x 256 up to 3 x 3 of 128 x 128, partial at the edges
SWITCH_K = (272, 16)                   # 9 TF32 / 5 f16 k-blocks; one partial k-block on both
PROBE_K = 1040                         # 33 TF32 / 17 f16 k-blocks, enough to separate the datapaths
SHARED = ("none", "a", "b", "a_nofit")  # a: A fits, B alternates; b: B fits, A alternates; a_nofit: every problem TF32
H100_SMS = 132                         # an H100 SXM; the GPU tests read the device's count


# ---- the schedule, restated --------------------------------------------------------------------------------------

def geometry(knobs):
    """(CTA group size, columns per tile, raster group in row tiles) of the wgmma kernel under `knobs`."""
    cg, bn = knobs.get("cta_group", 2), knobs.get("block_n", 256)
    return cg, bn, max(1, knobs.get("raster_rows", 2048) // (128 * cg))


def schedule(n, m, batch, knobs, sms):
    """Per CTA group, its tiles in order as (problem, row tile, column tile): tile t runs on group t mod G with
    G = min(tiles, SMs / CG); its problem is t / (tiles per problem), its place in the problem wgmma_tile_coord's."""
    cg, bn, raster = geometry(knobs)
    tr, tc = -(-n // (128 * cg)), -(-m // bn)
    per = tr * tc
    tiles = batch * per
    groups = min(tiles, sms // cg)
    return [[(t // per,) + fc.wgmma_tile_coord(t % per, tr, tc, raster) for t in range(g, tiles, groups)]
            for g in range(groups)]


def switches(sched, fits):
    """(groups that go from TF32 to f16, groups that go from f16 to TF32) between consecutive tiles."""
    up = down = 0
    for tiles in sched:
        seq = [fits[t[0]] for t in tiles]
        up += any(not x and y for x, y in zip(seq, seq[1:]))
        down += any(x and not y for x, y in zip(seq, seq[1:]))
    return up, down


def switch_batch(n, m, knobs, sms):
    """(batch, fits per problem): three waves of tiles, the problems of alternate waves fitting, so that a CTA group
    changes datapath from one of its tiles to the next."""
    cg, bn, _ = geometry(knobs)
    per = -(-n // (128 * cg)) * -(-m // bn)
    groups = sms // cg
    batch = -(-3 * groups // per)
    return batch, [(p * per // groups) % 2 == 0 for p in range(batch)]


# ---- data --------------------------------------------------------------------------------------------------------

def _plant_line(x, p, axis, value):
    """Scale (value None) or set one line of problem p: a row of A (axis 1) or a column of B (axis 2)."""
    n = x.shape[axis]
    i = (0, n // 2, n - 1)[p % 3]
    idx = (p, i, slice(None)) if axis == 1 else (p, slice(None), i)
    if value is None:
        x[idx] *= np.float32(tn.PLANT_SCALE)
    else:
        x[idx] = value


def mixed(a, b, fits, shared, plant=None):
    """Plant the lines that make problem p not fit where fits[p] is false: a row of A, or a column of B when A is
    shared; with `shared` "a_nofit" a row of the shared A, so that no problem fits.  plant None: times 2^20 (exact
    data); else the value to write (probe data).  In place; returns (a, b)."""
    if shared == "a_nofit":
        _plant_line(a, 0, 1, plant)
        return a, b
    for p, f in enumerate(fits):
        if not f:
            if shared == "a":
                _plant_line(b, p, 2, plant)
            else:
                _plant_line(a, p, 1, plant)
    return a, b


def expected_fits(shared, fits):
    return [False] * len(fits) if shared == "a_nofit" else list(fits)


def probe_operands(n, k, m, batch=1, seed=0, shared_a=False, shared_b=False):
    """Same-sign U[1, 10) rounded to half: the rounding to TF32 is the identity, every value a normal half."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(1, 10, ((1 if shared_a else batch), n, k)).astype(np.float16).astype(np.float32)
    b = rng.uniform(1, 10, ((1 if shared_b else batch), k, m)).astype(np.float16).astype(np.float32)
    return a, b


def _flags(mm, shared, transposed=False):
    return ((mm.FLAG_BATCH_SHARED_A if shared in ("a", "a_nofit") else 0)
            | (mm.FLAG_BATCH_SHARED_B if shared == "b" else 0) | (mm.FLAG_TRANSPOSED_A if transposed else 0))


def _a_in(a, transposed):
    return np.ascontiguousarray(np.swapaxes(a, -1, -2)) if transposed else a


# ---- the probe ---------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    return t


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _call(torch, mm, knobs, a, b, n, k, m, flags=0, batch=None):
    """C of one (batched) float call in a fresh context tuned with `knobs`, into a poisoned, guarded buffer."""
    with mm.Context(0) as ctx:
        ctx.set_tuning(**knobs)
        return tng._run(torch, mm, ctx, "tf32", tng._dev(torch, "tf32", a), tng._dev(torch, "tf32", b), n, k, m,
                        flags=flags, batch=batch)


def same_bits(x, y):
    return np.array_equal(np.asarray(x, np.float32).view(np.uint32), np.asarray(y, np.float32).view(np.uint32))


def classify(c, c_tf32):
    """The datapath a probe-data problem ran on, from its C and the same call's C under tf32_no_round = 1: "tf32"
    bit for bit equal, "tf32h" when fewer than half the elements agree, else "unclear"."""
    if same_bits(c, c_tf32):
        return "tf32"
    agree = np.asarray(c, np.float32).view(np.uint32) == np.asarray(c_tf32, np.float32).view(np.uint32)
    return "tf32h" if np.mean(agree) < 0.5 else "unclear"


def probe(torch, mm, knobs, a, b, n, k, m, flags=0, batch=None):
    """(C, the datapath of each problem as the probe sees it): the call under `knobs` and under `knobs` with
    tf32_no_round = 1, each in a fresh context."""
    c = _call(torch, mm, knobs, a, b, n, k, m, flags, batch)
    ct = _call(torch, mm, dict(knobs, tf32_no_round=1), a, b, n, k, m, flags, batch)
    if batch is None:
        return c, classify(c, ct)
    return c, [classify(c[i], ct[i]) for i in range(batch)]


def check_probe_datapaths(torch, mm, n=256, k=1024, m=256, knobs=None):
    """A fitting problem runs on f16, the same problem with one 2^16 in A (TF32-exact, not a half) on TF32."""
    a, b = probe_operands(n, k, m, seed=5)
    a, b = a[0], b[0]
    a_out = a.copy()
    a_out[n - 1, k - 1] = 2.0 ** 16
    assert tn.datapath(a, b) == "tf32h" and tn.datapath(a_out, b) == "tf32"
    c, path = probe(torch, mm, knobs or {}, a, b, n, k, m)
    assert path == "tf32h"
    tn.check_bound("tf32", c, *tn.prepared_product("tf32", a, b), k)
    assert probe(torch, mm, knobs or {}, a_out, b, n, k, m)[1] == "tf32"


def test_probe_separates_the_datapaths(torch, mm):
    check_probe_datapaths(torch, mm)
    check_probe_datapaths(torch, mm, 320, PROBE_K, 272, dict(cta_group=1, block_n=128))


# ---- 1. CTAs that switch datapath --------------------------------------------------------------------------------

def _switch_case(knobs, shared, k, sms, seed):
    """(a, b, batch, fits) of exact mixed data for one variant."""
    n, m = SWITCH_N, SWITCH_M
    batch, fits = switch_batch(n, m, knobs, sms)
    sa, sb = shared in ("a", "a_nofit"), shared == "b"
    a, b = tn.exact_operands("tf32h", n, k, m, batch, seed, sa, sb)
    return mixed(a, b, fits, shared) + (batch, expected_fits(shared, fits))


def _assert_datapaths(a, b, fits):
    for p, f in enumerate(fits):
        assert tn.datapath(a[p if a.shape[0] > 1 else 0], b[p if b.shape[0] > 1 else 0]) == ("tf32h" if f else "tf32")


def _exact_product(torch, a, b):
    """FP64 A B on the GPU: exact for the exact data."""
    t = lambda x: torch.from_numpy(np.asarray(x, np.float64)).cuda()
    return torch.matmul(t(a), t(b)).cpu().numpy()


@pytest.mark.parametrize("shared", SHARED)
@pytest.mark.parametrize("k", SWITCH_K)
@pytest.mark.parametrize("variant", VARIANTS, ids=[tng._vid(v) for v in VARIANTS])
def test_switching_ctas_exact(torch, mm, sms, variant, k, shared):
    knobs, transposed = variant
    n, m = SWITCH_N, SWITCH_M
    a, b, batch, fits = _switch_case(knobs, shared, k, sms, seed=61)
    _assert_datapaths(a, b, fits)
    if shared != "a_nofit":
        up, down = switches(schedule(n, m, batch, knobs, sms), fits)
        groups = len(schedule(n, m, batch, knobs, sms))
        assert up >= groups / 4 and down >= groups / 4, (up, down, groups)
    want = tn.store("tf32", _exact_product(torch, a, b))
    got = _call(torch, mm, knobs, _a_in(a, transposed), b, n, k, m, _flags(mm, shared, transposed), batch)
    for p in range(batch):
        tn.check_exact("tf32", got[p], want[p])


@pytest.mark.parametrize("shared", SHARED)
@pytest.mark.parametrize("variant", VARIANTS, ids=[tng._vid(v) for v in VARIANTS])
def test_switching_ctas_probe(torch, mm, sms, variant, shared):
    """Probe data: each problem of the batch equals its own single call bit for bit, and took its datapath."""
    knobs, transposed = variant
    n, k, m = SWITCH_N, PROBE_K, SWITCH_M
    batch, fits = switch_batch(n, m, knobs, sms)
    sa, sb = shared in ("a", "a_nofit"), shared == "b"
    a, b = mixed(*probe_operands(n, k, m, batch, 62, sa, sb), fits, shared, plant=np.float32(2.0 ** 16))
    fits = expected_fits(shared, fits)
    _assert_datapaths(a, b, fits)
    c, paths = probe(torch, mm, knobs, _a_in(a, transposed), b, n, k, m, _flags(mm, shared, transposed), batch)
    assert paths == [("tf32h" if f else "tf32") for f in fits], paths
    with mm.Context(0) as ctx:
        ctx.set_tuning(**knobs)
        for p in range(batch):
            ap, bp = _a_in(a[p if not sa else 0], transposed), b[p if not sb else 0]
            single = tng._run(torch, mm, ctx, "tf32", tng._dev(torch, "tf32", ap), tng._dev(torch, "tf32", bp), n, k,
                              m, flags=mm.FLAG_TRANSPOSED_A if transposed else 0)
            assert same_bits(c[p], single), p


# ---- 2. accumulate -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shared", ("none", "a", "b"))
@pytest.mark.parametrize("k", SWITCH_K)
@pytest.mark.parametrize("knobs", [{}, dict(cta_group=1, block_n=128, tma_store=0)],
                         ids=["default", "cg1_bn128_direct"])
def test_switching_ctas_accumulate_exact(torch, mm, sms, knobs, k, shared):
    """C_old = A B2 for B2 another draw of B with the same scales and plants: C_old + P = A (B + B2), an integer of at
    most 2^23 times the power of two of its row and column, exact in FP32."""
    n, m = SWITCH_N, SWITCH_M
    a, b, batch, fits = _switch_case(knobs, shared, k, sms, seed=63)
    _, b2, _, _ = _switch_case(knobs, shared, k, sms, seed=64)
    _assert_datapaths(a, b, fits)
    old = tn.store("tf32", _exact_product(torch, a, b2))
    want = tn.store("tf32", _exact_product(torch, a, b.astype(np.float64) + b2))
    assert np.array_equal(want, tn.store("tf32", _exact_product(torch, a, b)).astype(np.float64) + old)
    nbytes = old.nbytes
    raw = torch.full((nbytes + tng.GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
    c = raw[:nbytes].view(torch.float32)
    c.copy_(torch.from_numpy(old.reshape(-1)).cuda())
    with mm.Context(0) as ctx:
        ctx.set_tuning(**knobs)
        da, db = tng._dev(torch, "tf32", a), tng._dev(torch, "tf32", b)
        ctx.enqueue_accumulate(mm.FLOAT, mm.MULTIPLY, mm.ADD, da.data_ptr(), db.data_ptr(), c.data_ptr(), n, k, m,
                               batch, flags=_flags(mm, shared), stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    assert bool((raw[nbytes:] == 0xFF).all()), "the call wrote past C"
    got = c.cpu().numpy().reshape(batch, n, m)
    for p in range(batch):
        tn.check_exact("tf32", got[p], want[p])


# ---- 3. rounding boundaries on every preparation route ----------------------------------------------------------

# (float32 bits, the datapath its problem takes): 65520 rounds up to 2^16, 2^-14 (1 - 2^-12) up to 2^-14
BOUNDARY = {"65520": (0x477FF000, "tf32"), "65504": (0x477FE000, "tf32h"), "2^-14(1-2^-12)": (0x387FF000, "tf32h"),
            "2^-15": (0x38000000, "tf32"), "1e-40": (np.float32(1e-40).view(np.uint32), "tf32"),
            "-0": (0x80000000, "tf32h")}


def boundary_shape(sms):
    """n x k of A that round_tf32_kernel's grid (16 blocks of 256 threads per SM, one float4 each) covers in more than
    one pass; K = 1040 (16 k-tiles of 64 and a partial one)."""
    k = PROBE_K
    n = (16 * sms * 256 * 4) // k + 64
    return n + (-n) % 64 + 1, k, 192


@pytest.mark.parametrize("place", ["last", "tile_edge"])
@pytest.mark.parametrize("route", ["a", "at", "b"])
@pytest.mark.parametrize("value", sorted(BOUNDARY))
def test_rounding_boundary_sets_the_datapath(torch, mm, sms, value, route, place):
    """One value planted in A (row-major or stored K x N) or B, against a zero row of B (a zero column of A): C is the
    product of the rest.  The probe classifies the call; a 65520 sent to f16 would be inf there, and inf * 0 NaN."""
    bits, path = BOUNDARY[value]
    v = np.uint32(bits).view(np.float32)
    n, k, m = boundary_shape(sms)
    a, b = probe_operands(n, k, m, seed=65)
    a, b = a[0], b[0]
    assert n * k // 4 > 16 * sms * 256
    if route == "b":      # B is K x M in storage, transposed in 64 x 64 tiles
        i, j = (k - 1, m - 1) if place == "last" else (63, 127)
        b[i, j] = v
        a[:, i] = 0
    else:                 # A is N x K, or K x N in storage (FLAG_TRANSPOSED_A)
        si, sj = (k - 1, n - 1) if route == "at" else (n - 1, k - 1)
        if place == "tile_edge":
            si, sj = 63, 127
        i, j = (sj, si) if route == "at" else (si, sj)
        a[i, j] = v
        b[j, :] = 0
    assert tn.datapath(a, b) == path
    flags = mm.FLAG_TRANSPOSED_A if route == "at" else 0
    c, seen = probe(torch, mm, {}, _a_in(a, route == "at"), b, n, k, m, flags)
    assert not np.isnan(c).any()
    assert seen == path, (value, seen)


# ---- 4. fits words are per call ----------------------------------------------------------------------------------

PER_CALL = (256, PROBE_K, 256)


def _fit_and_not(n, k, m):
    """Probe data, and the same with 65520 against a zero row of B (runs on TF32; as f16 its C would hold NaN)."""
    a, b = probe_operands(n, k, m, seed=66)
    a, b = a[0], b[0]
    b[k - 1, :] = 0
    a_out = a.copy()
    a_out[n - 1, k - 1] = np.uint32(0x477FF000).view(np.float32)
    assert tn.datapath(a, b) == "tf32h" and tn.datapath(a_out, b) == "tf32"
    return a, a_out, b


def test_fits_words_reset_per_call(torch, mm):
    n, k, m = PER_CALL
    a, a_out, b = _fit_and_not(n, k, m)
    fresh = {}
    for name, x in (("fit", a), ("no fit", a_out)):
        fresh[name], path = probe(torch, mm, {}, x, b, n, k, m)
        assert path == ("tf32h" if name == "fit" else "tf32")
    with mm.Context(0) as ctx:
        for i, name in enumerate(["fit", "no fit", "fit", "no fit"]):
            got = tng._run(torch, mm, ctx, "tf32", tng._dev(torch, "tf32", a if name == "fit" else a_out),
                           tng._dev(torch, "tf32", b), n, k, m)
            assert same_bits(got, fresh[name]), (i, name)


def test_graph_replay_follows_operand_contents(torch, mm):
    """A call captured once, replayed after fitting, non-fitting and again fitting contents were copied into its
    operand buffers: a stale "fits" shows as NaN, a stale "does not fit" as TF32's bits."""
    n, k, m = PER_CALL
    a, a_out, b = _fit_and_not(n, k, m)
    fresh = {}
    for name, x in (("fit", a), ("no fit", a_out)):
        fresh[name], path = probe(torch, mm, {}, x, b, n, k, m)
        assert path == ("tf32h" if name == "fit" else "tf32")
    da, db = tng._dev(torch, "tf32", a), tng._dev(torch, "tf32", b)
    raw = torch.full((n * m * 4 + tng.GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
    c = raw[:n * m * 4].view(torch.float32)
    with mm.Context(0) as ctx:
        ctx.reserve(mm.FLOAT, n, k, m)
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            ctx.enqueue(mm.FLOAT, mm.MULTIPLY, mm.ADD, da.data_ptr(), db.data_ptr(), c.data_ptr(), n, k, m,
                        stream=s.cuda_stream)
        for i, name in enumerate(["fit", "no fit", "fit"]):
            da.copy_(torch.from_numpy(a if name == "fit" else a_out).cuda())
            raw[:n * m * 4].fill_(0xFF)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            got = c.cpu().numpy().reshape(n, m)
            assert bool((raw[n * m * 4:] == 0xFF).all()), "the replay wrote past C"
            assert not np.isnan(got).any(), (i, name)
            assert same_bits(got, fresh[name]), (i, name)
        del g
