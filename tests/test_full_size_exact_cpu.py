"""CPU checks of tests/test_full_size_exact_gpu.py's infrastructure (tests/full_size_check.py,
tensor_numerics.full_size_scheme): the exact data is exact by construction, the torch restatements of Naive<>'s
order equal the oracle bit for bit, and the comparison rejects a wrong, an unwritten and a guard-overwriting C with a
report that names the tile that wrote the element."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_size_check as fc  # noqa: E402
import tensor_numerics as tn  # noqa: E402

torch = pytest.importorskip("torch")

# (path, K) of every tensor-core case of the GPU file
WORKLOADS = [("tf32", 16384), ("tf32x3", 16384), ("f16", 32768), ("bf16", 32768), ("u8", 16384), ("dmma", 8192)]
# (largest finite, smallest normal) of each output type; float32 for the TF32 paths
_RANGE = {"tf32": (float(np.finfo(np.float32).max), 2.0 ** -126), "f16": (65504.0, 2.0 ** -14),
          "bf16": (float.fromhex("0x1.fep127"), 2.0 ** -126), "dmma": (float(np.finfo(np.float64).max), 2.0 ** -1022)}


@pytest.mark.parametrize("path,k", WORKLOADS, ids=["%s-%d" % w for w in WORKLOADS])
def test_full_size_scheme_is_exact_by_construction(path, k):
    """The bound follows from the magnitudes alone: limit^2 K within the path's exact accumulation, operands and C
    normal and finite in their types, and the exact C representable in float32 (the reference's middle step)."""
    lim, ea, eb = tn.full_size_scheme(path, k)
    s = lim * lim * k
    if path == "u8":
        assert lim == 255 and s < 2 ** 31
        return
    assert 1 <= lim <= tn.TYPE_INT_LIMIT[path]
    assert s <= tn.FULL_SIZE_S_LIMIT[path]
    if path != "dmma":
        assert s <= tn.EXACT_S_LIMIT and lim == tn.exact_limit(path, k)
    else:
        assert lim == 1024
    big, tiny = _RANGE["tf32" if path == "tf32x3" else path]
    (ea0, ea1), (eb0, eb1) = ea, eb
    # operands: every |x| in [2^e_lo, lim 2^e_hi], integers that the type's significand holds
    for e0, e1 in (ea, eb):
        assert 2.0 ** e0 >= tiny and lim * 2.0 ** e1 < big
    # C: an integer of magnitude <= s times 2^(ea + eb), every nonzero |C| at least that power of two
    c_max, c_min = s * 2.0 ** (ea1 + eb1), 2.0 ** (ea0 + eb0)
    assert c_max < big and c_min >= tiny
    if path == "f16":
        assert c_max < 2 ** 15 and c_min >= 2.0 ** -12
    if path != "dmma":
        assert s < 2 ** 24                      # the exact C fits float32's significand
        assert lim == {16384: 16, 32768: 11}[k]


def test_full_size_scheme_data_on_small_shapes():
    """exact_operands draws nonzero integers within the limit times the cycling row / column scales, and the
    FP64 reference is the exact product, stored in each output type."""
    n, k, m = 37, 64, 45
    for path in ("tf32h", "f16", "bf16", "dmma"):
        a, b = fc.exact_operands(torch, path, n, k, m, seed=3, device="cpu", row_block=16)
        lim, (ea0, ea1), (eb0, eb1) = tn.full_size_scheme(path, k)
        a64, b64 = a.to(torch.float64), b.to(torch.float64)
        ia = a64 / torch.exp2(ea0 + torch.arange(n, dtype=torch.float64) % (ea1 - ea0 + 1))[:, None]
        ib = b64 / torch.exp2(eb0 + torch.arange(m, dtype=torch.float64) % (eb1 - eb0 + 1))[None, :]
        for i in (ia, ib):
            assert bool((i == torch.round(i)).all()) and bool((i.abs() >= 1).all()) and int(i.abs().max()) <= lim
        want = fc.fp64_reference(torch, path, a, b, row_block=16)
        exact = (a64.numpy() @ b64.numpy())
        np.testing.assert_array_equal(want.to(torch.float64).numpy(), tn.to_float64(path, tn.store(path, exact)))
    # "tf32": the "tf32h" data with A's last row times 2^20; only that row of the exact C changes, by that power of two
    a, b = fc.exact_operands(torch, "tf32", n, k, m, seed=3, device="cpu", row_block=16)
    ah, bh = fc.exact_operands(torch, "tf32h", n, k, m, seed=3, device="cpu", row_block=16)
    assert torch.equal(b, bh) and torch.equal(a[:-1], ah[:-1]) and torch.equal(a[-1], ah[-1] * tn.PLANT_SCALE)
    assert tn.datapath(a.numpy(), b.numpy()) == "tf32" and tn.datapath(ah.numpy(), bh.numpy()) == "tf32h"
    want = fc.fp64_reference(torch, "tf32", a, b, row_block=16)
    exact = a.to(torch.float64).numpy() @ b.to(torch.float64).numpy()
    np.testing.assert_array_equal(want.to(torch.float64).numpy(), exact)
    a, b = fc.exact_operands(torch, "u8", n, k, m, seed=3, device="cpu")
    want = fc.fp64_reference(torch, "u8", a, b, row_block=16)
    exact = a.numpy().astype(np.int64) @ b.numpy().astype(np.int64)
    np.testing.assert_array_equal(want.numpy(), (exact % 256).astype(np.uint8))


# ---- the torch restatements of Naive<> ---------------------------------------------------------------------------

SHAPES = [(33, 320, 47), (5, 1024, 19), (1, 64, 1)]


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_min_plus_reference_equals_naive(oracle, shape):
    n, k, m = shape
    g = torch.Generator().manual_seed(11)
    a = torch.rand((n, k), generator=g) * 9.0 + 1.0
    b = torch.rand((k, m), generator=g) * 9.0 + 1.0
    got = fc.min_plus_reference(torch, a, b).numpy()
    want = oracle.naive(oracle.FLOAT, oracle.ADD, oracle.MIN, a.numpy(), b.numpy(), n, k, m)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_sequential_half_reference_equals_naive(oracle, shape):
    """half sums of U[0, 1) products reach hundreds at K = 1024, where every half addition rounds."""
    n, k, m = shape
    g = torch.Generator().manual_seed(12)
    a = torch.rand((n, k), generator=g).to(torch.float16)
    b = torch.rand((k, m), generator=g).to(torch.float16)
    got = fc.sequential_half_reference(torch, a, b).numpy()
    want = oracle.naive(oracle.HALF, oracle.MULTIPLY, oracle.ADD, a.numpy(), b.numpy(), n, k, m)
    assert got.tobytes() == want.tobytes()
    # not the FP64 product rounded once: the half accumulation is what is being restated
    assert got.tobytes() != (a.double() @ b.double()).half().numpy().tobytes() or k < 256


# ---- tile locations ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,m", [(16384, 16384), (32768, 32768), (2305, 4368), (8192, 1000)])
def test_wgmma_tile_index_inverts_the_schedule(n, m):
    """wgmma_tile_index is the inverse of the device's tile_coord over every tile, raster tail groups included."""
    tr, tc = math.ceil(n / fc.WGMMA_TILE), math.ceil(m / fc.WGMMA_TILE)
    seen = set()
    for t in range(tr * tc):
        r, c = fc.wgmma_tile_coord(t, tr, tc)
        assert 0 <= r < tr and 0 <= c < tc
        assert fc.wgmma_tile_index(r, c, tr, tc) == t
        seen.add((r, c))
    assert len(seen) == tr * tc


def test_float_16384_schedule_is_what_the_tests_claim():
    """4096 tiles on 66 CTA groups of an H100 (132 SMs): 62 or more tiles per group; the last tile's report."""
    loc = fc.wgmma_locator(16384, 16384, 132)
    msg = loc(16383, 16383)
    assert "persistent tile 4095 of 4096" in msg and "CTA group %d of 66" % (4095 % 66) in msg
    assert "its tile #62" in msg and "(row tile 63, column tile 63)" in msg
    assert fc.dmma_tile_rows(8192, 8192, 132) == 128 and fc.dmma_tile_rows(8192, 8192, 132, forced=64) == 64


# ---- the comparison rejects each defect and names the tile ---------------------------------------------------------

def _simulated(path, n, m, poison=0xFF):
    """A correct C with a poisoned guard after it, as the GPU tests hold them: (want, c, guard)."""
    dt = {"tf32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "u8": torch.uint8}[path]
    g = torch.Generator().manual_seed(5)
    want = (torch.randint(1, 200, (n, m), generator=g)).to(dt)
    nbytes = want.numel() * want.element_size()
    raw = torch.full((nbytes + fc.GUARD,), poison, dtype=torch.uint8)
    c = raw[:nbytes].view(dt).view(n, m)
    c.copy_(want)
    return want, c, raw[nbytes:]


N, M, BLOCK = 1000, 1100, 256   # row blocks [0, 256) ... [768, 1000): the last one is partial


@pytest.mark.parametrize("path", ["tf32", "f16", "bf16", "u8"])
def test_compare_accepts_a_correct_c(path):
    want, c, guard = _simulated(path, N, M)
    fc.check_guard(torch, path, guard, 0xFF)
    fc.compare(torch, path, c, want, fc.wgmma_locator(N, M, 132), "value", 0xFF, row_block=BLOCK)
    fc.compare(torch, path, c, lambda r0, r1: want[r0:r1], fc.wgmma_locator(N, M, 132), "bits", 0xFF,
               row_block=BLOCK)


@pytest.mark.parametrize("mode", ["value", "bits"])
@pytest.mark.parametrize("path", ["tf32", "f16", "bf16", "u8"])
def test_compare_rejects_one_wrong_element_in_the_last_row_block(path, mode):
    want, c, _ = _simulated(path, N, M)
    row, col = 997, 777            # wgmma tile (3, 3): 4 x 5 tiles, one raster group of 4: tile 3 * 4 + 3 = 15
    c[row, col] = c[row, col] + 1
    loc = fc.wgmma_locator(N, M, 132)
    with pytest.raises(AssertionError) as e:
        fc.compare(torch, path, c, want, loc, mode, 0xFF, row_block=BLOCK)
    msg = str(e.value)
    assert "1 of %d elements wrong (0 still hold" % (N * M) in msg
    assert "first at (row 997, col 777)" in msg
    assert "(row tile 3, column tile 3)" in msg and "persistent tile 15 of 20" in msg


@pytest.mark.parametrize("path", ["tf32", "f16", "bf16"])
def test_compare_rejects_one_element_still_holding_the_poison(path):
    """0xFF bytes are NaN in every float type: a never-written element equals nothing."""
    want, c, _ = _simulated(path, N, M)
    c.view(torch.uint8).view(N, M * c.element_size())[300, 5 * c.element_size():6 * c.element_size()] = 0xFF
    loc = fc.grid_locator("semiring_tile_kernel", 128, 128, N, M)
    for mode in ("value", "bits"):
        with pytest.raises(AssertionError) as e:
            fc.compare(torch, path, c, want, loc, mode, 0xFF, row_block=BLOCK)
        msg = str(e.value)
        assert "1 of %d elements wrong (1 still hold the poison byte 0xFF)" % (N * M) in msg
        assert "first at (row 300, col 5)" in msg and "blockIdx (x 0, y 2)" in msg


def test_compare_rejects_an_unwritten_uint8_element_under_one_of_the_two_poisons():
    """Every byte is a legal uint8 result, so the element left holding the poison passes under the poison equal to
    its right value and fails under the other one."""
    failures = 0
    for poison in (0x00, 0xFF):
        want, c, _ = _simulated("u8", N, M, poison)
        want[10, 20] = 0x00
        c[10, 20] = poison          # never written
        try:
            fc.compare(torch, "u8", c, want, fc.wgmma_locator(N, M, 132), "bits", poison, row_block=BLOCK)
        except AssertionError as e:
            failures += 1
            assert "first at (row 10, col 20)" in str(e) and "(row tile 0, column tile 0)" in str(e)
    assert failures == 1


@pytest.mark.parametrize("offset", [0, 1, fc.GUARD - 1])
def test_check_guard_rejects_one_changed_byte(offset):
    _, _, guard = _simulated("f16", 64, 64)
    guard[offset] = 0x7E
    with pytest.raises(AssertionError, match=r"wrote 1 of the 4096 guard bytes after C; first at byte \+%d: 0x7E"
                       % offset):
        fc.check_guard(torch, "f16", guard, 0xFF)


def test_dmma_and_semiring_reports_name_the_cta():
    loc = fc.grid_locator("gemm_dmma_tma_kernel", fc.dmma_tile_rows(8192, 8192, 132, forced=64), 128, 8192, 8192)
    assert "blockIdx (x 63, y 127) of a 64 x 128 grid of 64 x 128 tiles" in loc(8191, 8191)
    loc = fc.grid_locator("semiring_ring_kernel", 128, 128, 8192, 8192)
    assert "semiring_ring_kernel CTA blockIdx (x 2, y 1) of a 64 x 64 grid" in loc(200, 300)
