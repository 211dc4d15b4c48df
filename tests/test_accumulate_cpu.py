"""mm_kernel_enqueue_accumulate without a GPU: the restatement of R (tests/accumulate_naive.py) pinned on hand-picked
cases, and proof that the data of tests/test_accumulate_gpu.py rejects plausible wrong kernels.

The GPU tests hold C_new to R(C_old, P), P being the plain call's result on the same data.  Here P is Naive<> restated
by semiring_data.simulate (pinned to the oracle by tests/test_semiring_data_cpu.py), C_old is drawn exactly as the GPU
tests draw it, and each defect below must change C_new somewhere -- or be listed with the reason it cannot:
  ignored    C_old not read: C_new = P
  tile       one 128 x 128 tile of C left as P (every tile, in turn)
  swapped    R(P, C_old)
  seeded     the accumulators seeded with C_old instead of R in the epilogue
  flavour    float Min / Max with the other flavour (literal against FMNMX)
  twice      R(R(C_old, P), P)
  batch      another problem's C_old
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accumulate_naive as an  # noqa: E402
import bf16_naive  # noqa: E402
import semiring_data as sd  # noqa: E402
from semiring_data import ADD, AND, BF16, DOUBLE, FLOAT, FLOATING, HALF, INT32, MAX, MIN, MULTIPLY, UINT8  # noqa: E402

SEED = 7   # the GPU tests' seed for C_old


def _f(dtype, vals):
    return an._round(dtype, np.array(vals, dtype=np.float64))


# ---- the restatement on hand-picked cases ------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [FLOAT, DOUBLE, HALF, BF16])
def test_literal_min_max_signed_zero_ties_and_nan(dtype):
    pz, nz_, nan, one = _f(dtype, [0.0, -0.0, np.nan, 1.0])
    bits = an._bits
    for rd in (MIN, MAX):   # at a tie of +0 and -0 neither is below the other: both keep P
        assert bits(an.reduce_once(dtype, rd, nz_, pz)) == bits(pz)
        assert bits(an.reduce_once(dtype, rd, pz, nz_)) == bits(nz_)
        assert bits(an.reduce_once(dtype, rd, nan, one)) == bits(one)      # a NaN C_old gives P
        assert bits(an.reduce_once(dtype, rd, one, nan)) == bits(nan)      # a NaN P is kept


def test_fmnmx_signed_zero_and_nan():
    pz, nz_, nan, one = np.float32([0.0, -0.0, np.nan, 1.0])
    for c, p in ((nz_, pz), (pz, nz_)):
        assert an._bits(an.reduce_once(FLOAT, MIN, c, p, fmnmx=True)) == an._bits(nz_)
        assert an._bits(an.reduce_once(FLOAT, MAX, c, p, fmnmx=True)) == an._bits(pz)
    for rd in (MIN, MAX):
        assert an.reduce_once(FLOAT, rd, nan, one, fmnmx=True) == one
        assert an.reduce_once(FLOAT, rd, one, nan, fmnmx=True) == one
        assert np.isnan(an.reduce_once(FLOAT, rd, nan, nan, fmnmx=True))


@pytest.mark.parametrize("dtype", [FLOAT, DOUBLE, HALF, BF16])
def test_infinities_and_identities(dtype):
    inf, ninf, one, two = _f(dtype, [np.inf, -np.inf, 1.0, 2.0])
    assert np.isnan(an._value(dtype, an.reduce_once(dtype, ADD, inf, ninf)))
    assert an._value(dtype, an.reduce_once(dtype, ADD, inf, one)) == np.inf
    assert an._value(dtype, an.reduce_once(dtype, MULTIPLY, ninf, two)) == -np.inf
    big, tiny = sd.identity(dtype, MIN), sd.identity(dtype, MAX)
    assert an._bits(an.reduce_once(dtype, MIN, big, two)) == an._bits(two)      # Min's identity gives P
    assert an._bits(an.reduce_once(dtype, MAX, tiny, two)) == an._bits(two)
    assert an._bits(an.reduce_once(dtype, ADD, _f(dtype, [0.0])[0], two)) == an._bits(two)
    assert an._bits(an.reduce_once(dtype, AND, _f(dtype, [np.nan])[0], two)) == an._bits(one)   # NaN is nonzero
    assert an._bits(an.reduce_once(dtype, AND, _f(dtype, [-0.0])[0], two)) == an._bits(_f(dtype, [0.0])[0])


def test_integer_wrap():
    assert an.reduce_once(UINT8, ADD, np.uint8(200), np.uint8(100)) == 44
    assert an.reduce_once(UINT8, MULTIPLY, np.uint8(16), np.uint8(17)) == 16
    assert an.reduce_once(INT32, ADD, np.int32(2 ** 31 - 1), np.int32(1)) == -2 ** 31
    assert an.reduce_once(sd.UINT32, MULTIPLY, np.uint32(2 ** 31 + 1), np.uint32(3)) == (3 * (2 ** 31 + 1)) % 2 ** 32


def test_half_p_is_rounded_before_the_add():
    """a * b = 2^-11 (1 + 2^-11 - 2^-21) rounds to P = 2^-11; 1 + P is a tie and rounds to 1, where one rounding of
    1 + a*b would give 1 + 2^-10.  C_new is defined by P: 1."""
    a, b = np.float16(1 + 2.0 ** -10), np.float16(2.0 ** -11 * (1 - 2.0 ** -11))
    p = an.reduce_once(HALF, MULTIPLY, a, b)
    assert p == np.float16(2.0 ** -11)
    assert an.reduce_once(HALF, ADD, np.float16(1), p) == np.float16(1)
    assert np.float16(1.0 + float(a) * float(b)) == np.float16(1 + 2.0 ** -10)


def test_bf16_p_is_rounded_before_the_add():
    one = bf16_naive.from_double(np.array([1.0]))[0]
    p = bf16_naive.from_double(np.array([2.0 ** -8]))[0]                        # a tie at 1 (ulp 2^-7)
    assert bf16_naive.to_float(an.reduce_once(BF16, ADD, one, p)) == 1.0
    above = 2.0 ** -8 * (1 + 2.0 ** -9)                                         # rounds to 2^-8 as a bfloat16 P
    assert bf16_naive.from_double(np.array([above]))[0] == p
    assert bf16_naive.to_float(bf16_naive.from_double(np.array([1.0 + above])))[0] == 1 + 2.0 ** -7


@pytest.mark.parametrize("dtype,torch_name", [(HALF, "float16"), (BF16, "bfloat16")])
@pytest.mark.parametrize("reduce_op", [ADD, MULTIPLY])
def test_16_bit_arithmetic_against_torch(dtype, torch_name, reduce_op):
    """On values whose exact sum and product fit float32, torch-CPU's float32-then-round is one correct rounding."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    x = rng.uniform(0.0625, 2.0, size=4096) * rng.choice([-1, 1], size=4096)
    y = rng.uniform(0.0625, 2.0, size=4096) * rng.choice([-1, 1], size=4096)
    cx, cy = an._round(dtype, x), an._round(dtype, y)
    tdt = getattr(torch, torch_name)
    if dtype == BF16:
        tx = torch.from_numpy(cx.view(np.int16)).view(tdt)
        ty = torch.from_numpy(cy.view(np.int16)).view(tdt)
    else:
        tx, ty = torch.from_numpy(cx), torch.from_numpy(cy)
    tr = tx + ty if reduce_op == ADD else tx * ty
    want = tr.view(torch.int16).numpy().view(np.uint16) if dtype == BF16 else tr.numpy()
    assert an.same(dtype, an.reduce_once(dtype, reduce_op, cx, cy), want)


def test_c_old_holds_the_specials_and_ties():
    n, m, k = sd.gpu_shape(FLOAT)
    p = sd.simulate(FLOAT, ADD, MIN, *sd.discriminating(FLOAT, ADD, MIN, n, k, m, 1))
    c = an.c_old(FLOAT, MIN, p, SEED)
    assert np.isnan(c).any() and np.isinf(c).any() and (c == p).any()
    assert ((c == 0) & np.signbit(c)).any() and ((c == 0) & ~np.signbit(c)).any()
    assert (c == np.float32(np.finfo(np.float32).max)).any()


# ---- the GPU data rejects wrong kernels --------------------------------------------------------------------------

PAIRS = [(dt, mp, rd) for dt in sd.TYPES for rd in sd.OPS for mp in (ADD, MULTIPLY)] + \
    [(dt, mp, rd) for dt in sd.FLOATING for rd in (MIN, MAX) for mp in (MIN, MAX, AND)]
FMNMX = [(FLOAT, mp, rd) for mp in sd.OPS for rd in (MIN, MAX)]


def _seeded(dtype, map_op, reduce_op, a, b, c):
    """Naive<> with its accumulators seeded with C_old (the defect): R applied k times, starting from C_old."""
    ar = sd._Arith(dtype)
    av, bv = ar.load(a), ar.load(b)
    acc = ar.load(c).copy()
    for kk in range(av.shape[1]):
        acc = ar.apply(reduce_op, acc, ar.apply(map_op, av[:, kk:kk + 1], bv[kk:kk + 1, :]))
    return ar.store(acc)


def exempt(dtype, map_op, reduce_op, defect, fmnmx):
    """Why a defect cannot show, or None."""
    literal_minmax = reduce_op in (MIN, MAX) and not fmnmx
    if defect == "swapped" and not (literal_minmax and dtype in FLOATING):
        return "R is commutative here: only the literal floating Min / Max tell C_old from P (+-0 ties, NaN)"
    if defect == "seeded" and (dtype not in FLOATING or reduce_op == AND):
        return "R is associative and exact here: seeding the reduction with C_old gives the same result"
    if defect == "flavour" and reduce_op == MAX and (fmnmx or map_op == AND):
        # the flavours differ only at a +-0 tie and where P is NaN.  A Max's P is at least its identity
        # numeric_limits<float>::min() > 0, and is NaN only through a NaN term, which FMNMX never keeps and an And never
        # makes
        return "P >= FLT_MIN and never NaN here: fmaxf(c, p) and the literal Max agree on every c"
    if defect == "twice" and reduce_op in (MIN, MAX, AND):
        return "R is idempotent: R(R(c, p), p) = R(c, p)"
    return None


def _defects(dtype, map_op, reduce_op, fmnmx, a, b, p, c, want):
    n, m = p.shape
    yield "ignored", p
    for r0 in range(0, n, sd.TILE):
        for c0 in range(0, m, sd.TILE):
            got = want.copy()
            got[r0:r0 + sd.TILE, c0:c0 + sd.TILE] = p[r0:r0 + sd.TILE, c0:c0 + sd.TILE]
            yield "tile", got
    yield "swapped", an.reduce_once(dtype, reduce_op, p, c, fmnmx)
    if not fmnmx and map_op in (ADD, MULTIPLY):   # the other Maps' pairs are here for the flavour
        yield "seeded", _seeded(dtype, map_op, reduce_op, a, b, c)
    if dtype == FLOAT and reduce_op in (MIN, MAX):
        yield "flavour", an.reduce_once(dtype, reduce_op, c, p, not fmnmx)
    yield "twice", an.reduce_once(dtype, reduce_op, want, p, fmnmx)
    yield "batch", an.reduce_once(dtype, reduce_op, an.c_old(dtype, reduce_op, p, SEED + 1), p, fmnmx)


@pytest.mark.parametrize("dt,mp,rd,fmnmx", [x + (False,) for x in PAIRS] + [x + (True,) for x in FMNMX],
                         ids=lambda v: str(v))
def test_gpu_data_rejects_wrong_kernels(dt, mp, rd, fmnmx):
    n, m, k = sd.gpu_shape(dt)
    a, b = an.data(dt, mp, rd, n, k, m, 5, exact=not fmnmx)
    p = sd.simulate(dt, mp, rd, a, b)
    if fmnmx:   # the float default: Naive<> with FMNMX on NaN-free data equals the literal one
        assert not np.isnan(p).any()
    c = an.c_old(dt, rd, p, SEED)
    want = an.reduce_once(dt, rd, c, p, fmnmx)
    for defect, got in _defects(dt, mp, rd, fmnmx, a, b, p, c, want):
        reason = exempt(dt, mp, rd, defect, fmnmx)
        if reason is None:
            assert not an.same(dt, got, want, rd), "%s: the data does not reject '%s'" % (sd.pair_name(dt, mp, rd), defect)
        else:   # checked both ways: an exempt defect must really be invisible
            assert an.same(dt, got, want, rd), "%s: '%s' is exempt (%s) but shows" % (sd.pair_name(dt, mp, rd), defect,
                                                                                reason)
