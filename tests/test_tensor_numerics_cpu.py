"""CPU tests of tests/tensor_numerics.py and of the power of tests/test_tensor_numerics_gpu.py's checks.

* `rna_tf32` and `split_tf32` pinned against hand-written bit patterns and identities.
* The exact-data generators' precondition (S <= 2^22, values exact and normal in the type) for every shape the GPU
  file runs.
* Power: each GPU check runs here on simulated kernels over a smaller version of the same data (same K, same
  generator).  A correct kernel (FP32 accumulation of the prepared operands in a random order, rounding to nearest
  and toward zero) must pass every check; each wrong kernel must be rejected by the check named for it:

  | wrong kernel                                    | rejected by                                                  |
  |-------------------------------------------------|--------------------------------------------------------------|
  | TF32 operands truncated, not rounded, one side  | identity product of that route; TF32 tie data; the K = 544    |
  |                                                 | same-sign bound                                              |
  | round to nearest even instead of rna            | identity product (tie patterns); TF32 tie data               |
  | one 32-element k-block dropped in one tile      | multi-wave exact product                                     |
  | two adjacent C columns swapped in 16 rows       | multi-wave exact product                                     |
  | one output tile left unwritten                  | poison check (uint8_t: the exact product under two poisons)  |
  | f16 accumulating in half                        | multi-wave exact product (f16); long-K same-sign bound (f16) |
  | 3xTF32 without lo_a * hi_b / hi_a * lo_b        | 3xTF32 identity product, A route / B route                   |
  | preparation before the saturating round_tf32    | special values: TF32 and 3xTF32 near-overflow operands       |
  | 3xTF32 split before lo = 0 / hi' for infinities | special values: 3xTF32 infinite operands                     |

  The long-K bound is too loose to catch a one-sided truncation (it biases each product by about 2^-12 relative,
  inside alpha * 16384 * 2^-23 S); the identity and tie checks catch it exactly.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tensor_numerics as tn  # noqa: E402
import test_tensor_numerics_gpu as gpu  # noqa: E402  (shapes and data of the GPU checks; no GPU is touched)


def f32(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


def bits(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


# ---- rna_tf32 ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("x,want", [
    (0x3F801000, 0x3F802000), (0xBF801000, 0xBF802000),     # ties: away from zero, both signs
    (0x3F803000, 0x3F804000), (0xBF803000, 0xBF804000),     # ties with an odd kept bit: also away from zero
    (0x3F800FFF, 0x3F800000), (0x3F801001, 0x3F802000),     # just below / above half
    (0x3FFFF000, 0x40000000), (0xBFFFF000, 0xC0000000),     # carry into the exponent
    (0x7F7FE000, 0x7F7FE000), (0x7F7FEFFF, 0x7F7FE000),     # the largest TF32, and below its half-way point
    (0x7F7FF000, 0x7F7FE000), (0x7F7FF800, 0x7F7FE000), (0x7F7FFFFF, 0x7F7FE000), (0xFF7FFFFF, 0xFF7FE000),
    (0x00000000, 0x00000000), (0x80000000, 0x80000000),     # signed zeros
    (0x7F800000, 0x7F800000), (0xFF800000, 0xFF800000),     # infinities
    (0x00800000, 0x00800000),                               # smallest normal
    (0x007FF000, 0x00800000),                               # subnormal rounding up into the smallest normal
    (0x00001000, 0x00002000), (0x80000FFF, 0x80000000),     # subnormal tie, subnormal rounding to -0
])
def test_rna_tf32_bit_patterns(x, want):
    assert int(bits(tn.rna_tf32(f32([x])))[0]) == want


def test_rna_tf32_band_below_flt_max_saturates_and_bare_instruction_overflows():
    band = f32(np.arange(0x7F7FF000, 0x80000000, 1, dtype=np.uint32)[:0x1000])
    assert np.all(bits(tn.rna_tf32(band)) == 0x7F7FE000)
    assert np.all(bits(tn.rna_tf32(-band)) == 0xFF7FE000)
    assert np.all(np.isposinf(tn.rna_tf32(band, saturate=False)))
    below = f32(np.arange(0x7F7FE000, 0x7F7FF000, dtype=np.uint32))
    assert np.all(bits(tn.rna_tf32(below)) == 0x7F7FE000)


def test_rna_tf32_nan_stays_nan():
    nans = f32([0x7FC00000, 0x7F800001, 0xFFFFFFFF, 0x7FBFFFFF])
    assert np.all(np.isnan(tn.rna_tf32(nans)))


def test_rna_tf32_is_nearest_with_ties_away_on_random_patterns():
    x = tn.tf32_patterns(1, 1 << 16)
    r = tn.rna_tf32(x).astype(np.float64)
    x64 = x.astype(np.float64)
    assert np.all(bits(r.astype(np.float32)) & 0x1FFF == 0)
    ulp = np.exp2(np.floor(np.log2(np.abs(x64))) - 10)
    fine = np.abs(x64) < tn.FLT_MAX * (1 - 2.0 ** -12)        # below the saturating band
    assert np.all(np.abs(r - x64)[fine] <= ulp[fine] / 2)
    tie = (bits(x) & 0x1FFF) == 0x1000
    assert np.all((np.abs(r) > np.abs(x64))[tie & fine])      # ties away from zero


# ---- split_tf32 --------------------------------------------------------------------------------------------------

def test_split_tf32_parts_are_tf32_and_sum_to_x():
    x = np.concatenate([tn.tf32_patterns(2, 1 << 17, min_exp=24),
                        f32(np.arange(0x7F000000, 0x7F7FFFFF, 0x3F1, dtype=np.uint32))])   # the top binade
    hi, lo = tn.split_tf32(x)
    assert np.all(bits(hi) & 0x1FFF == 0) and np.all(bits(lo) & 0x1FFF == 0)
    assert np.all(np.isfinite(hi)) and np.all(np.isfinite(lo))
    with np.errstate(over="ignore"):
        s = (hi.astype(np.float64) + lo).astype(np.float32).astype(np.float64)
    x64 = x.astype(np.float64)
    fin = np.isfinite(s)
    assert np.count_nonzero(~fin) <= 8                        # hi + lo rounds past FLT_MAX only at its very top
    assert np.all(np.abs(s - x64)[fin] <= 2.0 ** -22 * np.abs(x64[fin]))


def test_split_tf32_infinities_and_nan():
    hi, lo = tn.split_tf32(f32([0x7F800000, 0xFF800000, 0x7FC00000, 0x7F7FFFFF]))
    assert np.isposinf(hi[0]) and np.isneginf(hi[1]) and lo[0] == 0 and lo[1] == 0
    assert np.isnan(hi[2]) and np.isnan(lo[2])
    assert bits(hi[3:])[0] == 0x7F7FE000 and np.isfinite(lo[3])
    assert np.all(tn.finite_or_zero(hi[:2]) == 0) and np.isnan(tn.finite_or_zero(hi[2:3]))[0]


# ---- generators --------------------------------------------------------------------------------------------------

def _gpu_exact_shapes():
    """Every exact case of the GPU file; the f16-datapath float data ("tf32h") last, after the cases of the other
    paths in their own order."""
    cases = []
    for last in (False, True):
        keep = lambda p: (p == "tf32h") == last
        cases += [(p, s, 1) for p, s in gpu.MULTIWAVE.items() if keep(p)]
        cases += [(p, (1, w, w), 1) for p, w in gpu.WIDTH.items() if keep(p)]
        cases += [(p, (129, 3 * w, 17 * w), 1) for p, w in gpu.WIDTH.items() if keep(p)]
        cases += [(p, s, 9) for p, s in gpu.BATCHED.items() if keep(p)]
    return cases


@pytest.mark.parametrize("path,shape,batch", _gpu_exact_shapes())
def test_exact_generator_precondition(path, shape, batch):
    n, k, m = shape
    w = gpu.WIDTH[path]
    assert k % w == 0 and m % w == 0
    if path == "u8":
        assert k * 255 * 255 < 2 ** 31                    # the integer accumulator never wraps
        return
    lim = tn.exact_limit(path, k)
    assert k * lim * lim <= tn.EXACT_S_LIMIT and lim <= tn.TYPE_INT_LIMIT[path]
    a, b = tn.exact_operands(path, min(n, 40), k, min(m, 48), batch, seed=1)
    a64, b64 = tn.to_float64(path, a), tn.to_float64(path, b)
    # every value an integer up to lim times a power of two, held exactly by the input type
    for x in (a64, b64):
        e = np.floor(np.log2(np.abs(x)))
        frac = np.abs(x) / np.exp2(e)
        assert np.all(frac * 2 ** 12 == np.round(frac * 2 ** 12))
    if path in tn.FLOAT_PATHS:
        assert np.array_equal(tn.rna_tf32(a), a) and np.array_equal(tn.split_tf32(b)[1], np.zeros_like(b))
    s_int = np.abs(np.round(a64 / _row_scale(a64))) @ np.abs(np.round(b64 / _col_scale(b64)))
    assert s_int.max() <= tn.EXACT_S_LIMIT


def _row_scale(a):
    return np.exp2(np.floor(np.log2(np.abs(a).min(axis=-1, keepdims=True))))


def _col_scale(b):
    return np.exp2(np.floor(np.log2(np.abs(b).min(axis=-2, keepdims=True))))


def test_tie_data_separates_rounding_modes():
    for route in ("a", "b"):
        a, b = tn.tie_operands(route, 129, 64, 272, seed=24)
        x = a if route == "a" else b
        assert np.all(bits(x) & 0x1FFF == 0x1000)           # every value of that operand is a TF32 tie
        assert np.mean(tn.rna_tf32(x) != tn.rne_tf32(x)) > 0.4
        assert np.all(tn.rna_tf32(x) != tn.trunc_tf32(x))


# ---- simulated kernels ------------------------------------------------------------------------------------------

def _round32(s, mode):
    f = s.astype(np.float32)
    if mode == "rz":
        with np.errstate(invalid="ignore"):
            over = np.abs(f.astype(np.float64)) > np.abs(s)
        f = np.where(over, np.nextafter(f, np.float32(0)), f)
    return f


def simulate(path, ap, bp, mode="rn", seed=0, half_accumulate=False, skip=None):
    """C of a kernel that accumulates the prepared operands' products one by one in a random order of k, in FP32
    rounding to nearest ("rn") or toward zero ("rz") (in half with half_accumulate), then stores C in the output
    type.  skip(kk) -> boolean mask of C elements that drop product kk."""
    ap, bp = np.asarray(ap, np.float64), np.asarray(bp, np.float64)
    order = np.random.default_rng(seed).permutation(ap.shape[1])
    if path == "dmma":
        acc = np.zeros((ap.shape[0], bp.shape[1]))
    else:
        acc = np.zeros((ap.shape[0], bp.shape[1]), np.float16 if half_accumulate else np.float32)
    with np.errstate(all="ignore"):
        for kk in order:
            p = ap[:, kk:kk + 1] * bp[kk:kk + 1, :]
            if skip is not None:
                p = np.where(skip(kk), 0.0, p)
            s = acc.astype(np.float64) + p
            if path == "dmma":
                acc = s
            elif half_accumulate:
                acc = s.astype(np.float16)
            else:
                acc = _round32(s, mode)
    if path == "u8":
        return np.mod(acc.astype(np.float64), 256).astype(np.uint8)
    return tn.store(path, acc.astype(np.float64))


MODES = ("rn", "rz")


# identity products -----------------------------------------------------------------------------------------------

def _identity_sim(path, route, drop=None):
    """Prepared operands of the GPU identity case (the transposed route stores A differently, same values) and its
    expected C.  drop: a 3xTF32 block of K' left out."""
    a, b, n, k, m, want = gpu._identity_case(path, route, rows=128)
    ap, bp = tn.prepared_operands(path, a, b)
    if drop is not None:
        ap = ap.copy()
        ap[:, drop * k:(drop + 1) * k] = 0
    return ap, bp, want


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("path,route", gpu.IDENTITY_CASES)
def test_identity_check_accepts_correct_kernels(path, route, mode):
    ap, bp, want = _identity_sim(path, route)
    tn.check_exact(path, simulate(path, ap, bp, mode), want)


@pytest.mark.parametrize("route", ["a", "at", "b"])
@pytest.mark.parametrize("wrong", ["trunc", "rne"])
def test_identity_check_rejects_wrong_tf32_rounding(route, wrong):
    f = tn.trunc_tf32 if wrong == "trunc" else tn.rne_tf32   # the identity side is unchanged by any rounding
    a, b, _, _, _, want = gpu._identity_case("tf32", route, rows=128)
    ap, bp = f(a).astype(np.float64), f(b).astype(np.float64)
    with pytest.raises(AssertionError):
        tn.check_exact("tf32", simulate("tf32", ap, bp), want)


@pytest.mark.parametrize("route,term", [("a", 2), ("b", 1)])
def test_identity_check_rejects_3xtf32_missing_cross_term(route, term):
    """A' = [hi | hi' | lo]: block 2 is lo_a * hi_b (seen on the A route), block 1 hi_a * lo_b (seen on the B route)."""
    ap, bp, want = _identity_sim("tf32x3", route, drop=term)
    with pytest.raises(AssertionError):
        tn.check_exact("tf32x3", simulate("tf32x3", ap, bp), want)


# TF32 ties -------------------------------------------------------------------------------------------------------

def _tie_case(route, prep_a=tn.rna_tf32, prep_b=tn.rna_tf32):
    n, k, m = 24, 64, 32                               # the GPU test's K; fewer rows and columns
    a, b = tn.tie_operands(route, n, k, m, seed=24)
    want = tn.store("tf32", tn.rna_tf32(a).astype(np.float64) @ tn.rna_tf32(b).astype(np.float64))
    return prep_a(a).astype(np.float64), prep_b(b).astype(np.float64), want


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("route", ["a", "b"])
def test_tie_check_accepts_correct_kernels(route, mode):
    ap, bp, want = _tie_case(route)
    tn.check_exact("tf32", simulate("tf32", ap, bp, mode), want)


@pytest.mark.parametrize("route", ["a", "b"])
@pytest.mark.parametrize("wrong", ["trunc", "rne"])
def test_tie_check_rejects_wrong_rounding_on_one_side(route, wrong):
    f = tn.trunc_tf32 if wrong == "trunc" else tn.rne_tf32
    ap, bp, want = _tie_case(route, **({"prep_a": f} if route == "a" else {"prep_b": f}))
    with pytest.raises(AssertionError):
        tn.check_exact("tf32", simulate("tf32", ap, bp), want)


# multi-wave exact products -----------------------------------------------------------------------------------------

def _exact_sim_case(path, batch=1):
    n, k, m = gpu.MULTIWAVE[path]
    a, b = tn.exact_operands(path, 48, k, 64, batch, seed=21)
    ap, bp = tn.prepared_operands(path, a[0], b[0])
    want = tn.store(path, tn.to_float64(path, a[0]) @ tn.to_float64(path, b[0]))
    return ap, bp, want


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("path", sorted(gpu.MULTIWAVE))
def test_exact_check_accepts_correct_kernels(path, mode):
    ap, bp, want = _exact_sim_case(path)
    tn.check_exact(path, simulate(path, ap, bp, mode, seed=3), want)


@pytest.mark.parametrize("path", sorted(gpu.MULTIWAVE))
def test_exact_check_rejects_a_dropped_k_block(path):
    ap, bp, want = _exact_sim_case(path)
    rows, cols = np.arange(want.shape[0])[:, None] < 128, np.arange(want.shape[1])[None, :] < 256   # one tile
    c = simulate(path, ap, bp, skip=lambda kk: (32 <= kk < 64) & rows & cols)
    with pytest.raises(AssertionError):
        tn.check_exact(path, c, want)


@pytest.mark.parametrize("path", sorted(gpu.MULTIWAVE))
def test_exact_check_rejects_swapped_columns(path):
    ap, bp, want = _exact_sim_case(path)
    c = simulate(path, ap, bp).copy()
    c[16:32, [6, 7]] = c[16:32, [7, 6]]
    with pytest.raises(AssertionError):
        tn.check_exact(path, c, want)


@pytest.mark.parametrize("path", sorted(gpu.MULTIWAVE))
def test_poison_check_rejects_an_unwritten_tile(path):
    """Floats: poison 0xFF (NaN) is never a result.  uint8_t: every byte is, so the GPU test runs with poison 0x00
    and 0xFF and requires the exact result both times; a block left unwritten fails at least one of the two."""
    ap, bp, want = _exact_sim_case(path)
    c = np.ascontiguousarray(simulate(path, ap, bp))
    failures = 0
    for poison in ((0x00, 0xFF) if path == "u8" else (0xFF,)):
        if path != "u8":
            tn.check_no_poison(c.view(np.uint8), c.itemsize, poison)
        raw = c.view(np.uint8).reshape(c.shape[0], -1).copy()
        raw[:16, : 32 * c.itemsize] = poison              # one 16 x 32 epilogue block never stored
        if path != "u8":
            with pytest.raises(AssertionError):
                tn.check_no_poison(raw, c.itemsize, poison)
        try:
            tn.check_exact(path, raw.view(c.dtype).reshape(c.shape), want)
        except AssertionError:
            failures += 1
    assert failures >= 1


def test_exact_check_rejects_half_accumulation():
    ap, bp, want = _exact_sim_case("f16")
    with pytest.raises(AssertionError):
        tn.check_exact("f16", simulate("f16", ap, bp, half_accumulate=True), want)


def test_batched_generator_gives_each_problem_its_own_scale():
    for path in sorted(gpu.BATCHED):
        a, b = tn.exact_operands(path, 8, gpu.BATCHED[path][1], 64, 9, seed=25)
        want = tn.store(path, np.matmul(tn.to_float64(path, a), tn.to_float64(path, b)))
        assert all(not np.array_equal(want[i], want[i + 1]) for i in range(8))


# error bounds ----------------------------------------------------------------------------------------------------

# the GPU shapes, fewer rows and columns: K decides the bound
BOUND_SIM_SHAPES = {"513x544x544": (6, 544, 8), "128x16384x256": (2, 16384, 4)}


def _bound_sim(path, kind, shape, **kw):
    n, k, m = BOUND_SIM_SHAPES[shape]
    a, b = tn.bound_operands(path, kind, n, k, m, seed=5)
    ap, bp = tn.prepared_operands(path, a, b)
    r, s = ap @ bp, np.abs(ap) @ np.abs(bp)
    return simulate(path, ap, bp, **kw), r, s, k


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", sorted(BOUND_SIM_SHAPES))
@pytest.mark.parametrize("kind", tn.BOUND_KINDS)
@pytest.mark.parametrize("path", gpu.BOUND_PATHS)
def test_bound_accepts_correct_kernels(path, kind, shape, mode):
    if path == "dmma" and mode == "rz":
        pytest.skip("DMMA rounds to nearest in FP64")
    c, r, s, k = _bound_sim(path, kind, shape, mode=mode, seed=7)
    tn.check_bound(path, c, r, s, k)


@pytest.mark.parametrize("side", ["a", "b"])
def test_short_k_bound_rejects_one_sided_truncation(side):
    """At K = 544 on same-sign data the bias of a truncated operand (about 2^-12 of S) exceeds alpha K 2^-23 S."""
    n, k, m = BOUND_SIM_SHAPES["513x544x544"]
    a, b = tn.bound_operands("tf32", "same_sign", n, k, m, seed=5)
    ap, bp = tn.prepared_operands("tf32", a, b)
    r, s = ap @ bp, np.abs(ap) @ np.abs(bp)
    if side == "a":
        ap = tn.trunc_tf32(a).astype(np.float64)
    else:
        bp = tn.trunc_tf32(b).astype(np.float64)
    with pytest.raises(AssertionError):
        tn.check_bound("tf32", simulate("tf32", ap, bp), r, s, k)


def test_long_k_bound_rejects_half_accumulation():
    c, r, s, k = _bound_sim("f16", "same_sign", "128x16384x256", half_accumulate=True)
    with pytest.raises(AssertionError):
        tn.check_bound("f16", c, r, s, k)


# special values -----------------------------------------------------------------------------------------------------

def _prefix_operands(path, a, b):
    """The preparation before the saturating round_tf32 and the infinity rules of the 3xTF32 split."""
    def split(x):
        hi = tn.rna_tf32(x, saturate=False)
        with np.errstate(invalid="ignore"):
            lo = tn.rna_tf32((x - hi).astype(np.float32), saturate=False)
        return hi, lo
    if path == "tf32":
        return tn.rna_tf32(a, saturate=False).astype(np.float64), tn.rna_tf32(b, saturate=False).astype(np.float64)
    ha, la = split(a)
    hb, lb = split(b)
    return (np.concatenate([ha, ha, la], axis=1).astype(np.float64),
            np.concatenate([hb, lb, hb], axis=0).astype(np.float64))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("path", ["tf32", "tf32x3", "f16", "bf16", "dmma"])
def test_special_value_checks_accept_correct_kernels(path, mode):
    a, b = tn.special_operands(path, seed=26)
    ap, bp = tn.prepared_operands(path, a, b)
    ref = tn.ieee_reference(ap, bp)
    s = tn.ieee_reference(np.abs(ap), np.abs(bp))
    c = simulate(path, ap, bp, mode if path != "dmma" else "rn", seed=4)
    tn.check_classes(path, c, ref)
    fin = tn.value_class(ref) == 0
    tn.check_bound(path, c[fin], ref[fin], s[fin], 64)


@pytest.mark.parametrize("what", ["infinity", "near_overflow"])
@pytest.mark.parametrize("path", ["tf32", "tf32x3"])
def test_special_value_check_rejects_the_old_preparation(path, what):
    """The preparation before the fix: cvt.rna overflowing to inf, and lo = inf - inf = NaN.  TF32 fails on the
    near-overflow operands only; 3xTF32 on both."""
    a, b = tn.special_operands(path, seed=26)
    ap, bp = tn.prepared_operands(path, a, b)
    ref = tn.ieee_reference(ap, bp)
    rows, cols = np.indices(ref.shape)
    finite = tn.value_class(ref) == 0
    if what == "infinity":       # non-finite C away from the near-overflow rows (16..23) and columns (50..53)
        keep = ~finite & (rows < 16) & (cols < 48)
    else:                        # finite C in the near-overflow rows and columns
        keep = finite & (((rows >= 16) & (rows < 24)) | ((cols >= 50) & (cols < 54)))
    assert keep.sum() > 8
    oa, ob = _prefix_operands(path, a, b)
    c = simulate(path, oa, ob)
    if path == "tf32" and what == "infinity":
        tn.check_classes(path, c[keep], ref[keep])         # infinities were already right on the single pass
        return
    with pytest.raises(AssertionError):
        tn.check_classes(path, c[keep], ref[keep])
