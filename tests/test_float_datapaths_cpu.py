"""CPU tests of the data, the schedule restatement and the checks of tests/test_float_datapaths_gpu.py and of the
two float datapaths in tests/test_tensor_numerics_gpu.py: each generator gives the datapath its key names, the planted
data stays exact, the chosen batches really switch datapath on every CTA group schedule, and the checks reject numpy
models of a kernel that takes the wrong datapath.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_size_check as fc  # noqa: E402
import tensor_numerics as tn  # noqa: E402
import test_float_datapaths_gpu as fd  # noqa: E402  (shapes and data of the GPU checks; no GPU is touched)
import test_tensor_numerics_gpu as tng  # noqa: E402

SMS = fd.H100_SMS


# ---- generators name their datapath -------------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["tf32", "tf32h"])
def test_exact_data_takes_the_datapath_of_its_key(path):
    for n, k, m in (tng.MULTIWAVE[path], (1, 16, 16), (129, 48, 272)):
        for plant in ("first", "last"):
            a, b = tn.exact_operands(path, min(n, 40), k, min(m, 48), seed=1, plant=plant)
            assert tn.datapath(a[0], b[0]) == path
    n, k, m = tng.BATCHED[path]
    for sa, sb in ((False, False), (True, False), (False, True)):
        a, b = tn.exact_operands(path, 24, k, 32, 9, 25, sa, sb)
        assert all(tn.datapath(a[0 if sa else i], b[0 if sb else i]) == path for i in range(9))
        if path == "tf32":    # one row per copy of A: first and last alternating, the last copy's last row
            big = [np.flatnonzero(np.abs(x).min(axis=1) >= 2.0 ** 16).tolist() for x in a]
            assert big == [[r] for r in tn.plant_rows("tf32", 24, a.shape[0])]
            assert big == [[0]] if a.shape[0] == 1 else (big[0] == [0] and big[-1] == [23])


def test_plant_rows():
    assert tn.plant_rows("tf32h", 8, 3) == [None] * 3
    assert tn.plant_rows("tf32", 8, 1) == [0] and tn.plant_rows("tf32", 8, 1, "last") == [7]
    assert tn.plant_rows("tf32", 8, 4) == [0, 7, 0, 7] and tn.plant_rows("tf32", 8, 3) == [0, 7, 7]


@pytest.mark.parametrize("shared", fd.SHARED)
@pytest.mark.parametrize("variant", fd.VARIANTS[:8], ids=[tng._vid(v) for v in fd.VARIANTS[:8]])
def test_mixed_batches_take_the_datapaths_of_their_pattern(variant, shared):
    knobs, _ = variant
    batch, fits = fd.switch_batch(fd.SWITCH_N, fd.SWITCH_M, knobs, SMS)
    sa, sb = shared in ("a", "a_nofit"), shared == "b"
    want = fd.expected_fits(shared, fits)
    assert (not any(want)) if shared == "a_nofit" else (any(want) and not all(want))
    a, b = tn.exact_operands("tf32h", 8, 16, 8, batch, 1, sa, sb)
    fd._assert_datapaths(*fd.mixed(a, b, fits, shared), want)
    a, b = fd.probe_operands(8, 32, 8, batch, 1, sa, sb)
    fd._assert_datapaths(*fd.mixed(a, b, fits, shared, plant=np.float32(2.0 ** 16)), want)


@pytest.mark.parametrize("value", sorted(fd.BOUNDARY))
def test_boundary_values_round_across_the_fits_boundary(value):
    bits, path = fd.BOUNDARY[value]
    v = np.uint32(bits).view(np.float32).reshape(1)
    assert tn.datapath(v, np.float32([1.0])) == path
    rounded = float(tn.rna_tf32(v)[0])
    if value == "1e-40":      # a float subnormal stays one
        assert 0 < rounded < 2.0 ** -126
        return
    assert rounded == {"65520": 2.0 ** 16, "65504": 65504.0, "2^-14(1-2^-12)": 2.0 ** -14, "2^-15": 2.0 ** -15,
                       "-0": 0.0}[value]
    if value in ("65520", "2^-14(1-2^-12)"):
        assert rounded != float(v[0])     # the rounding, not the stored value, decides


def test_boundary_shape_takes_more_than_one_grid_stride_pass():
    n, k, m = fd.boundary_shape(SMS)
    assert n * k // 4 > 16 * SMS * 256 and n % 64 == 1 and k > 1024 and n > 64 and m > 128


# ---- exactness with the plants -------------------------------------------------------------------------------------

def _exact_int(a, b):
    """A B over the integers: every value an integer times a power of two >= 2^-10, scaled to exact int64."""
    s = 2.0 ** 10
    ai, bi = (a.astype(np.float64) * s).astype(np.int64), (b.astype(np.float64) * s).astype(np.int64)
    assert np.array_equal(ai / s, a) and np.array_equal(bi / s, b)
    return np.matmul(ai, bi), s * s


@pytest.mark.parametrize("shared", fd.SHARED)
@pytest.mark.parametrize("k", fd.SWITCH_K)
def test_planted_mixed_data_is_exact_in_fp32(k, shared):
    """C and C_old + P (the accumulate test) computed over the integers are float32 values."""
    knobs = {}
    a, b, batch, fits = fd._switch_case(knobs, shared, k, SMS, seed=63)
    _, b2, _, _ = fd._switch_case(knobs, shared, k, SMS, seed=64)
    a, b, b2 = a[:, :40], b[..., :48], b2[..., :48]
    for bb in (b, b + b2.astype(np.float64)):
        c, scale = _exact_int(a, bb)
        assert np.array_equal(c.astype(np.float32).astype(np.int64), c)          # exact in float32
        assert np.abs(c).max() / scale < 2.0 ** 60
    c, scale = _exact_int(a, b)
    assert np.array_equal(tn.store("tf32", np.matmul(a.astype(np.float64), b)).astype(np.float64) * scale, c)


@pytest.mark.parametrize("path", ["tf32", "tf32h"])
def test_batched_and_multiwave_exact_data_is_exact_in_fp32(path):
    for n, k, m, batch in ((40,) + tng.MULTIWAVE[path][1:2] + (48, 1), (24,) + tng.BATCHED[path][1:2] + (32, 9)):
        a, b = tn.exact_operands(path, n, k, m, batch, seed=2)
        c, scale = _exact_int(a, b)
        assert np.array_equal(c.astype(np.float32).astype(np.int64), c)
        assert np.array_equal(tn.store(path, np.matmul(a.astype(np.float64), b.astype(np.float64))) * scale, c)


# ---- the schedule --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", fd.VARIANTS, ids=[tng._vid(v) for v in fd.VARIANTS])
def test_schedule_restatement_covers_every_tile_once(variant):
    knobs, _ = variant
    cg, bn, raster = fd.geometry(knobs)
    n, m = fd.SWITCH_N, fd.SWITCH_M
    batch, _ = fd.switch_batch(n, m, knobs, SMS)
    sched = fd.schedule(n, m, batch, knobs, SMS)
    tr, tc = -(-n // (128 * cg)), -(-m // bn)
    assert len(sched) == min(batch * tr * tc, SMS // cg)
    seen = [t for tiles in sched for t in tiles]
    assert sorted(seen) == [(p, r, c) for p in range(batch) for r in range(tr) for c in range(tc)]
    per = tr * tc
    for g, tiles in enumerate(sched):
        for j, (p, r, c) in enumerate(tiles):
            assert p * per + fc.wgmma_tile_index(r, c, tr, tc, raster) == g + j * len(sched)


@pytest.mark.parametrize("variant", fd.VARIANTS, ids=[tng._vid(v) for v in fd.VARIANTS])
def test_every_variant_switches_a_quarter_of_the_groups_both_ways(variant):
    knobs, _ = variant
    n, m = fd.SWITCH_N, fd.SWITCH_M
    batch, fits = fd.switch_batch(n, m, knobs, SMS)
    sched = fd.schedule(n, m, batch, knobs, SMS)
    up, down = fd.switches(sched, fits)
    assert up >= len(sched) / 4 and down >= len(sched) / 4


def test_k_block_counts_differ_between_the_datapaths():
    kb = lambda k_bytes: -(-k_bytes // 128)
    assert (kb(272 * 4), kb(272 * 2)) == (9, 5) and (kb(16 * 4), kb(16 * 2)) == (1, 1)
    assert (kb(fd.PROBE_K * 4), kb(fd.PROBE_K * 2)) == (33, 17)


# ---- the checks reject a kernel on the wrong datapath -------------------------------------------------------------

def test_exact_check_rejects_a_non_fitting_problem_run_from_fp16_copies():
    """The fp16 copy of a row times 2^20 is +-inf: C holds inf or NaN there."""
    a, b = tn.exact_operands("tf32", 24, 272, 32, seed=3)
    a, b = a[0], b[0]
    want = tn.store("tf32", a.astype(np.float64) @ b.astype(np.float64))
    with np.errstate(over="ignore", invalid="ignore"):
        a16, b16 = tn.rna_tf32(a).astype(np.float16), tn.rna_tf32(b).astype(np.float16)
        wrong = tn.store("tf32", tn.ieee_reference(a16, b16))
    assert not np.isfinite(wrong[0]).all()
    tn.check_exact("tf32", tn.store("tf32", tn.ieee_reference(tn.rna_tf32(a), tn.rna_tf32(b))), want)
    with pytest.raises(AssertionError):
        tn.check_exact("tf32", wrong, want)


def test_boundary_check_rejects_65520_run_from_its_fp16_copy():
    """65520 rounds to 2^16: its fp16 copy is inf, and inf times the zero row of B is NaN in C."""
    a, b = fd.probe_operands(8, 64, 8, seed=4)
    a, b = a[0], b[0]
    a[7, 63], b[63, :] = np.uint32(0x477FF000).view(np.float32), 0
    with np.errstate(over="ignore", invalid="ignore"):
        wrong = tn.ieee_reference(tn.rna_tf32(a).astype(np.float16), b.astype(np.float16))
    assert np.isnan(wrong).any() and not np.isnan(tn.ieee_reference(tn.rna_tf32(a), b)).any()


def _sequential_fp32(a, b):
    """A TF32-datapath model: each element summed in k order in float32."""
    c = np.zeros((a.shape[0], b.shape[1]), np.float32)
    for kk in range(a.shape[1]):
        c = (c + np.float32(a[:, kk:kk + 1]) * b[kk:kk + 1, :]).astype(np.float32)
    return c


def test_probe_rejects_a_fitting_problem_run_on_tf32():
    """Modelled bits: a fitting problem computed as TF32 is bit for bit its tf32_no_round result, so the probe calls
    it "tf32"; a datapath that rounds its partial sums differently (here: once, from FP64) is called "tf32h"."""
    a, b = fd.probe_operands(16, fd.PROBE_K, 16, seed=6)
    a, b = a[0], b[0]
    tf32 = _sequential_fp32(a, b)
    other = (a.astype(np.float64) @ b.astype(np.float64)).astype(np.float32)
    assert fd.classify(tf32, tf32) == "tf32"
    assert fd.classify(other, tf32) == "tf32h"
    near = tf32.copy()
    near.view(np.uint32)[:4] ^= 1                        # a few last bits off: neither datapath
    assert fd.classify(near, tf32) == "unclear"
