"""Test infrastructure: what the tensor-core GEMMs compute, restated in numpy.

* Operand preparation bit for bit: `rna_tf32` is the device's `round_tf32` (cvt.rna.tf32.f32: round to nearest
  TF32, ties away from zero, a finite input saturating to +-0x7F7FE000 instead of overflowing), `split_tf32` the
  3xTF32 hi / lo split.  `prepared_operands` gives the operands a kernel actually multiplies.
* Exact data: integers scaled by a power of two per row of A, per column of B and per problem of a batch, with
  S = sum |a| |b| <= 2^22 over the integers.  Every product and every partial sum is then an integer times one
  power of two below 2^22, exact in FP32 in any order, with 2 bits to spare for any alignment truncation inside
  the tensor core.  The expected C is the exact value stored once in the output type.
* `check_bound`: the per-element error bound of the FP32-accumulating paths against an FP64 evaluation of the
  prepared operands, and of DMMA against an FP64 reference that carries error itself.
* `ieee_reference`: an elementwise FP64 evaluation (no BLAS, which may skip zero multipliers and hide inf * 0).

Paths: "tf32", "tf32h", "tf32x3", "f16", "bf16", "dmma" (double), "u8".  bfloat16 values are np.uint16 bit patterns.
"tf32" and "tf32h" are float (Multiply, Add) on its two datapaths: a problem whose TF32-rounded A and B all fit a half
(`fits_half`, gemm_hls_b200/csrc/fits_half.h) runs on the f16 wgmma, any other on TF32.  They share the type, the
preparation and the bound; only the exact data differs: "tf32h" fits, and "tf32" is the same data with one row of A
per problem times 2^20 (`PLANT_SCALE`), which no half holds.
"""
import math

import numpy as np

import bf16_naive

PATHS = ("tf32", "tf32h", "tf32x3", "f16", "bf16", "dmma", "u8")
FLOAT_PATHS = ("tf32", "tf32h", "tf32x3")
TF32_MAX_BITS = 0x7F7FE000          # the largest finite TF32 value (10 explicit mantissa bits)
FLT_MAX = float(np.finfo(np.float32).max)

# Integer magnitudes that the input type holds exactly, and that leave TF32 rounding the identity (so lo = 0).
TYPE_INT_LIMIT = {"tf32": 1024, "tf32h": 1024, "tf32x3": 1024, "f16": 2048, "bf16": 256, "dmma": 1024}
EXACT_S_LIMIT = 2 ** 22

# alpha_path of check_bound: |c - r| <= half an ulp + alpha * K_eff * 2^-23 * S.  alpha = 1 bounds any order of
# FP32 additions rounding toward zero.  Each value has >= 4x headroom over the worst alpha an H100 (80GB HBM3,
# 700 W power limit, 2026-10-16) needed over tests/test_tensor_numerics_gpu.py's bound cases (U[0.5, 1), N(0, 1),
# exponent-spread data at (513, 544, 544), (128, 16384, 256) and the multi-wave shape), and is above what a
# simulated round-toward-zero accumulation in random order needs (<= 0.19 on same-sign data,
# tests/test_tensor_numerics_cpu.py).  Worst seen on the H100, all on same-sign data:
#   tf32 0.0654, tf32x3 0.0416, f16 0.0534, bf16 0.0391.
ALPHA = {"tf32": 0.3, "tf32h": 0.3, "tf32x3": 0.25, "f16": 0.25, "bf16": 0.25}

# One row of A per problem of "tf32" exact data is scaled by this: its values are >= 2^16, TF32-exact but no half, so
# the problem runs on TF32.  Every C element of that row is still one integer <= 2^22 times one power of two (<= 2^41),
# exact in FP32; sent to the f16 datapath by mistake, the row's fp16 copy is +-inf and C holds inf or NaN there.
PLANT_SCALE = 2.0 ** 20


# ---- operand preparation --------------------------------------------------------------------------------------

def rna_tf32(x, saturate=True):
    """float32 -> float32 rounded to nearest TF32 (ties away from zero), as cvt.rna.tf32.f32.  `saturate`: a finite
    input whose rounding overflows becomes +-0x7F7FE000 (the library's round_tf32); False is the bare instruction.
    Subnormals round like normals (a carry out of the mantissa gives the smallest normal); +-0 and +-inf stay;
    NaN stays NaN (payload not modelled)."""
    u = np.array(x, dtype=np.float32).view(np.uint32)
    mag = u & np.uint32(0x7FFFFFFF)
    special = mag >= np.uint32(0x7F800000)
    r = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    if saturate:
        over = ~special & ((r & np.uint32(0x7FFFFFFF)) == np.uint32(0x7F800000))
        r = np.where(over, (r & np.uint32(0x80000000)) | np.uint32(TF32_MAX_BITS), r)
    return np.where(special, u, r).astype(np.uint32).view(np.float32)


def trunc_tf32(x):
    """The low 13 bits dropped: what tf32 wgmma reads from an unprepared float (a wrong preparation)."""
    u = np.array(x, dtype=np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32)


def rne_tf32(x):
    """Round to nearest TF32, ties to even (a wrong preparation: the device rounds ties away from zero)."""
    u = np.array(x, dtype=np.float32).view(np.uint32)
    r = (u + np.uint32(0xFFF) + ((u >> np.uint32(13)) & np.uint32(1))) & np.uint32(0xFFFFE000)
    return np.where((u & np.uint32(0x7FFFFFFF)) >= np.uint32(0x7F800000), u, r).astype(np.uint32).view(np.float32)


def split_tf32(x):
    """(hi, lo) of the 3xTF32 split: hi = rna(x), lo = rna(x - hi) (x - hi is exact in FP32), lo = 0 for +-inf."""
    x = np.asarray(x, dtype=np.float32)
    hi = rna_tf32(x)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = rna_tf32((x - hi).astype(np.float32))
    return hi, np.where(np.isinf(x), np.float32(0), lo).astype(np.float32)


def fits_half_each(x):
    """Elementwise gemm_hls_b200/csrc/fits_half.h on rna_tf32(x): the rounded value is +-0 or a normal half
    (2^-14 <= |v| < 2^16, biased float exponent 113 .. 142)."""
    u = rna_tf32(x).view(np.uint32)
    e = (u >> np.uint32(23)) & np.uint32(0xFF)
    return ((u & np.uint32(0x7FFFFFFF)) == 0) | ((e >= 113) & (e <= 142))


def fits_half(x):
    """Whether an operand sends its float problem to the f16 datapath: every TF32-rounded value is +-0 or a normal
    half.  A problem runs on f16 when both its A and its B fit."""
    return bool(np.all(fits_half_each(x)))


def datapath(a, b):
    """"tf32h" when the float problem (a, b) runs on the f16 wgmma, "tf32" when it runs on TF32."""
    return "tf32h" if fits_half(a) and fits_half(b) else "tf32"


def finite_or_zero(hi):
    """The hi of the 3xTF32 cross terms: +-inf replaced by 0, so that hi * hi alone carries infinities."""
    return np.where(np.isinf(hi), np.float32(0), hi).astype(np.float32)


def to_float64(path, x):
    """Values of an input or output array of `path` as float64 (bfloat16 from its bit patterns)."""
    if path == "bf16":
        return bf16_naive.to_float(x).astype(np.float64)
    return np.asarray(x).astype(np.float64)


def prepared_operands(path, a, b, transposed_a=False):
    """(A', B') in float64: the operands the kernel multiplies, C = A' B' accumulated.  a is n x k (k x n when
    transposed_a), b is k x m.  3xTF32 returns K' = 3K: A' = [hi | hi' | lo], B' = [hi ; lo ; hi'] with
    hi' = finite_or_zero(hi), i.e. hi_a hi_b + hi_a lo_b + lo_a hi_b."""
    a = np.asarray(a)
    if transposed_a:
        a = a.T
    if path in ("tf32", "tf32h"):
        return rna_tf32(a).astype(np.float64), rna_tf32(b).astype(np.float64)
    if path == "tf32x3":
        ha, la = split_tf32(a)
        hb, lb = split_tf32(b)
        ap = np.concatenate([ha, finite_or_zero(ha), la], axis=1).astype(np.float64)
        bp = np.concatenate([hb, lb, finite_or_zero(hb)], axis=0).astype(np.float64)
        return ap, bp
    return to_float64(path, a), to_float64(path, b)


def prepared_product(path, a, b, transposed_a=False, matmul=None):
    """(R, S): the FP64 product of the prepared operands and S = |A'| |B'|.  `matmul` (float64 arrays -> float64
    array) lets a caller run the two products elsewhere, e.g. on the GPU."""
    ap, bp = prepared_operands(path, a, b, transposed_a)
    mul = matmul or (lambda x, y: x @ y)
    return mul(ap, bp), mul(np.abs(ap), np.abs(bp))


def k_eff(path, k):
    return 3 * k if path == "tf32x3" else k


def ieee_reference(ap, bp):
    """sum_k ap[i, k] * bp[k, j] elementwise in float64 with IEEE inf / NaN semantics (small shapes only)."""
    with np.errstate(all="ignore"):
        return (np.asarray(ap, np.float64)[:, :, None] * np.asarray(bp, np.float64)[None, :, :]).sum(axis=1)


# ---- output types ---------------------------------------------------------------------------------------------

# (mantissa bits, smallest normal exponent) of each path's output type
_OUT_FORMAT = {"tf32": (23, -126), "tf32h": (23, -126), "tf32x3": (23, -126), "f16": (10, -14), "bf16": (7, -126),
               "dmma": (52, -1022)}


def half_ulp(path, x):
    """Half an ulp of the output type at |x| (float64), with the subnormal quantum as the floor."""
    mant, emin = _OUT_FORMAT[path]
    with np.errstate(divide="ignore"):
        e = np.maximum(np.floor(np.log2(np.abs(np.asarray(x, np.float64)))), emin)
    return np.exp2(e - mant - 1)


def store(path, exact):
    """The exact float64 C stored once in the output type (round to nearest even), as the kernel's epilogue does;
    uint8: modulo 256."""
    exact = np.asarray(exact, np.float64)
    if path in FLOAT_PATHS:
        return exact.astype(np.float32)
    if path == "f16":
        return exact.astype(np.float16)
    if path == "bf16":
        return bf16_naive.from_double(exact)
    if path == "dmma":
        return exact
    return np.mod(exact, 256).astype(np.uint8)


# ---- checks ---------------------------------------------------------------------------------------------------

def check_exact(path, c, want):
    """Every element equal to the exact expectation: bit-identical up to the sign of zero (a zero sum's sign is
    not pinned), no NaN anywhere.  Returns the number of mismatches (0) so that callers can assert on it."""
    c = np.asarray(c).reshape(-1)
    want = np.asarray(want).reshape(-1)
    if path == "u8":
        bad = int(np.count_nonzero(c != want))
    else:
        bad = int(np.count_nonzero(~(to_float64(path, c) == to_float64(path, want))))
    assert bad == 0, "%s: %d of %d elements differ from the exact product" % (path, bad, c.size)
    return bad


def check_no_poison(c_bytes, itemsize, poison):
    """No element of C (raw bytes) still holds the poison pattern the buffer was filled with."""
    b = np.asarray(c_bytes, dtype=np.uint8).reshape(-1, itemsize)
    left = int(np.count_nonzero((b == poison).all(axis=1)))
    assert left == 0, "%d elements of C were never written" % left
    return left


def gamma(path, k):
    if path == "dmma":
        return 2.0 * (k + 1) * 2.0 ** -53
    return ALPHA[path] * k_eff(path, k) * 2.0 ** -23


def check_bound(path, c, r, s, k):
    """|c - r| <= half_ulp(|r| + g S) + g S per element, g = gamma(path, k); r, s from prepared_product.
    Returns (worst |c - r| / bound, worst alpha observed): alpha_seen = max (|c - r| - half_ulp) / (K_eff 2^-23 S),
    the alpha the data needed (0 for DMMA)."""
    c = to_float64(path, c).reshape(np.shape(r))
    r = np.asarray(r, np.float64)
    s = np.asarray(s, np.float64)
    g = gamma(path, k)
    h = half_ulp(path, np.abs(r) + g * s)
    err = np.abs(c - r)
    bound = h + g * s
    ok = err <= bound
    if not bool(ok.all()):
        i = int(np.argmin(np.where(ok, 1, 0).reshape(-1)))
        raise AssertionError("%s: %d elements outside the bound; first at flat %d: c=%r r=%r S=%r bound=%r" % (
            path, int((~ok).sum()), i, c.reshape(-1)[i], r.reshape(-1)[i], s.reshape(-1)[i], bound.reshape(-1)[i]))
    worst = float(np.max(err / bound))
    alpha_seen = 0.0
    if path != "dmma":
        with np.errstate(divide="ignore", invalid="ignore"):
            a = np.maximum(err - h, 0) / (k_eff(path, k) * 2.0 ** -23 * s)
        alpha_seen = float(np.max(np.where(s > 0, a, 0)))
    return worst, alpha_seen


def value_class(x):
    """0 finite, 1 +inf, 2 -inf, 3 NaN."""
    x = np.asarray(x, np.float64)
    return np.where(np.isnan(x), 3, np.where(x == np.inf, 1, np.where(x == -np.inf, 2, 0)))


def check_classes(path, c, ref):
    """Class of every element (NaN, +inf, -inf, finite) equal to the IEEE reference's."""
    got, want = value_class(to_float64(path, c)).reshape(-1), value_class(ref).reshape(-1)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%s: %d elements of the wrong class, first at flat %d: got %d want %d" % (
        path, bad.size, bad[0], got[bad[0]], want[bad[0]])
    return 0


# ---- data -----------------------------------------------------------------------------------------------------

# exponent ranges of the per-row, per-column and per-problem scales; half shifts A down so that |C| < 2^15
_ROW_EXP, _COL_EXP, _PROB_EXP = (-3, -1), (-2, 0), (-1, 0)
_A_SHIFT = {"f16": -6}


def exact_limit(path, k):
    """Largest integer magnitude of the exact data at this K: k * limit^2 <= 2^22, within the type's exact range."""
    return min(TYPE_INT_LIMIT[path], int(math.isqrt(EXACT_S_LIMIT // k)))


# Exact data at the benchmark sizes (tests/test_full_size_exact_gpu.py): nonzero integers in [-limit, limit] times
# 2^ea per row of A and 2^eb per column of B, ea and eb cycling through these inclusive ranges.  Every C element is
# then an integer of magnitude <= limit^2 K times the one power of two 2^(ea + eb) of its row and column.  half:
# |C| <= 2^22 2^(-4 - 3) < 2^15, and every nonzero |C| >= 2^(-6 - 6) = 2^-12, a normal half.
_FULL_SIZE_EXP = {"tf32": ((-3, -1), (-2, 0)), "tf32h": ((-3, -1), (-2, 0)), "tf32x3": ((-3, -1), (-2, 0)),
                  "f16": ((-6, -4), (-6, -3)), "bf16": ((-3, -1), (-2, 0)), "dmma": ((-3, -1), (-2, 0))}
# Bound on limit^2 K: the FP32-accumulating paths keep 2 bits of FP32's 24 to spare (EXACT_S_LIMIT); DMMA
# accumulates in FP64 and keeps the same 2 bits of FP64's 53, so it takes the type's whole exact range (1024).
FULL_SIZE_S_LIMIT = {"tf32": EXACT_S_LIMIT, "tf32h": EXACT_S_LIMIT, "tf32x3": EXACT_S_LIMIT, "f16": EXACT_S_LIMIT,
                     "bf16": EXACT_S_LIMIT, "dmma": 2 ** 51}


def full_size_scheme(path, k):
    """(limit, (ea_lo, ea_hi), (eb_lo, eb_hi)) of the exact data of `path` at inner extent k: the largest integer
    magnitude with limit^2 k <= FULL_SIZE_S_LIMIT[path] within the type's exact range, and the exponent ranges of
    the row scales of A and the column scales of B.  uint8: (255, None, None), full-range bytes, whose products and
    sums are exact in the 32-bit accumulator (255^2 k < 2^31)."""
    if path == "u8":
        return 255, None, None
    lim = min(TYPE_INT_LIMIT[path], int(math.isqrt(FULL_SIZE_S_LIMIT[path] // k)))
    ea, eb = _FULL_SIZE_EXP[path]
    return lim, ea, eb


def _nonzero_ints(rng, lim, shape):
    return rng.integers(1, lim + 1, size=shape) * rng.choice(np.array([-1, 1]), size=shape)


def _in_dtype(path, x):
    if path in FLOAT_PATHS:
        return x.astype(np.float32)
    if path == "f16":
        return x.astype(np.float16)
    if path == "bf16":
        return bf16_naive.from_double(x)
    return x.astype(np.float64)


def plant_rows(path, n, copies, first="first"):
    """The row of each of A's copies that "tf32" data scales by PLANT_SCALE (None for every other path): copy 0 at
    its first row (`first` "first") or its last ("last"), then alternating, and in a batch the last copy always at
    its last row."""
    if path != "tf32":
        return [None] * copies
    rows = [0 if (i % 2 == 0) == (first == "first") else n - 1 for i in range(copies)]
    if copies > 1:
        rows[-1] = n - 1
    return rows


def exact_operands(path, n, k, m, batch=1, seed=0, shared_a=False, shared_b=False, plant="first"):
    """A (batch_a x n x k) and B (batch_b x k x m) of exact data for `path`, in its input type (batch_x = 1 when
    shared).  uint8: full-range bytes (the integer accumulation is exact for any data).  Asserts the exactness
    precondition S <= 2^22 (over the integers) and that every value and every C is a normal number of the type.
    "tf32": one row of each copy of A times PLANT_SCALE (plant_rows, `plant` the first copy's row), so that every
    problem runs on TF32; "tf32h": the same data without it, every problem on f16 (both asserted with fits_half)."""
    rng = np.random.default_rng(seed)
    ba, bb = (1 if shared_a else batch), (1 if shared_b else batch)
    if path == "u8":
        return (rng.integers(0, 256, size=(ba, n, k), dtype=np.uint8),
                rng.integers(0, 256, size=(bb, k, m), dtype=np.uint8))
    lim = exact_limit(path, k)
    assert k * lim * lim <= EXACT_S_LIMIT and lim <= TYPE_INT_LIMIT[path]
    ia, ib = _nonzero_ints(rng, lim, (ba, n, k)), _nonzero_ints(rng, lim, (bb, k, m))
    # distinct neighbours: adjacent rows / columns / problems never share a scale
    ea = _ROW_EXP[0] + (np.arange(n) * 2) % (_ROW_EXP[1] - _ROW_EXP[0] + 1) + _A_SHIFT.get(path, 0)
    eb = _COL_EXP[0] + np.arange(m) % (_COL_EXP[1] - _COL_EXP[0] + 1)
    ep = _PROB_EXP[0] + np.arange(batch) % (_PROB_EXP[1] - _PROB_EXP[0] + 1)
    # the problem's scale rides on A, or on B when A is shared, so that the problems of a batch still differ
    pa = ep[:ba, None, None] if not shared_a else np.zeros((1, 1, 1))
    pb = ep[:bb, None, None] if shared_a else np.zeros((1, 1, 1))
    a = ia * np.exp2(ea[None, :, None] + pa)
    b = ib * np.exp2(eb[None, None, :] + pb)
    emin = _ROW_EXP[0] + _COL_EXP[0] + _PROB_EXP[0] + _A_SHIFT.get(path, 0)
    emax = _ROW_EXP[1] + _COL_EXP[1] + _PROB_EXP[1] + _A_SHIFT.get(path, 0)
    if path == "f16":   # every operand and every C a normal half
        assert EXACT_S_LIMIT * 2.0 ** emax < 65504 and emin >= -14
        assert np.abs(a).min() >= 2.0 ** -14 and np.abs(b).min() >= 2.0 ** -14
    for i, r in enumerate(plant_rows(path, n, ba, plant)):
        if r is not None:
            a[i, r, :] *= PLANT_SCALE
    a, b = _in_dtype(path, a), _in_dtype(path, b)
    if path in ("tf32", "tf32h"):
        assert all(datapath(a[i if ba > 1 else 0], b[i if bb > 1 else 0]) == path for i in range(batch))
    return a, b


def tie_operands(route, n, k, m, seed=0):
    """TF32 tie data: odd integers in (2048, 4096) are exactly halfway between two TF32 values (rna rounds them away
    from zero, rne and truncation may not), times a power of two per row / column; the other operand holds small
    integers with k * 4096 * 16 <= 2^22, so that the product of the rounded operands is exact.  route "a": ties in
    A; "b": ties in B.  float32 A (n x k), B (k x m)."""
    rng = np.random.default_rng(seed)
    lim = EXACT_S_LIMIT // (k * 4096)
    assert lim >= 1
    ties = lambda shape: (2 * rng.integers(1024, 2048, size=shape) + 1) * rng.choice(np.array([-1, 1]), size=shape)
    small = lambda shape: _nonzero_ints(rng, lim, shape)
    ea = -3 + np.arange(n) % 4
    eb = -2 + np.arange(m) % 3
    ia, ib = (ties((n, k)), small((k, m))) if route == "a" else (small((n, k)), ties((k, m)))
    return (ia * np.exp2(ea[:, None])).astype(np.float32), (ib * np.exp2(eb[None, :])).astype(np.float32)


BOUND_KINDS = ("same_sign", "mixed", "spread")


def bound_operands(path, kind, n, k, m, seed=0):
    """Random data for check_bound, in the input type of `path`: "same_sign" U[0.5, 1), "mixed" N(0, 1), "spread"
    N(0, 1) times 2^e per row of A and per column of B, e uniform in [-20, 20] ([-2, 2] for half, which keeps C
    within half's range up to K = 16384)."""
    rng = np.random.default_rng(seed)
    if kind == "same_sign":
        a, b = rng.uniform(0.5, 1.0, (n, k)), rng.uniform(0.5, 1.0, (k, m))
    else:
        a, b = rng.standard_normal((n, k)), rng.standard_normal((k, m))
        if kind == "spread":
            w = 2 if path == "f16" else 20
            a = a * np.exp2(rng.integers(-w, w + 1, size=(n, 1)))
            b = b * np.exp2(rng.integers(-w, w + 1, size=(1, m)))
    return _in_dtype(path, a), _in_dtype(path, b)


# the largest finite value of each input type and its bit pattern family: near-overflow operands of the special test
_BIG = {"tf32": [np.uint32(0x7F7FF000), np.uint32(0x7F7FF800), np.uint32(0x7F7FFFFF), np.uint32(0x7F7FE000)],
        "f16": [65504.0, 65472.0], "bf16": [0x7F7F, 0x7F7E], "dmma": [np.finfo(np.float64).max, 1.5e308]}


def special_operands(path, n=64, k=64, m=64, seed=0):
    """Finite mixed-sign data with |x| in [0.5, 2), plus +-inf and NaN at chosen places of A and B, and near-overflow
    values of the type meeting B (or A) entries of 2^-10, so that their exact C is finite.  Input type of `path`."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0.5, 2.0, (n, k)) * rng.choice([-1.0, 1.0], (n, k))
    b = rng.uniform(0.5, 2.0, (k, m)) * rng.choice([-1.0, 1.0], (k, m))
    inf, nan = np.inf, np.nan
    a[1, 3], a[2, 5], a[4, 7] = inf, -inf, nan
    a[8, 20], a[8, 21] = inf, -inf                  # inf - inf in some columns, same-sign infinities in others
    b[9, 10], b[11, 12], b[13, 14] = -inf, inf, nan
    b[3, 40] = inf                                  # meets A's +inf at (1, 3): +-inf, never NaN
    # near overflow: A[r, 30] big against B[30, :] = +-2^-10 x, B[40, 50] big against A[:, 40] = +-2^-10 x
    b[30, :] = np.sign(b[30, :]) * np.exp2(-10) * rng.uniform(0.5, 1.0, m)
    a[:, 40] = np.sign(a[:, 40]) * np.exp2(-10) * rng.uniform(0.5, 1.0, n)
    out_a, out_b = _in_dtype(path, a), _in_dtype(path, b)
    big = _BIG["tf32" if path in ("tf32", "tf32x3") else path]
    for i, r in enumerate(range(16, 16 + 2 * len(big))):
        v, sign = big[i % len(big)], (-1) ** i
        if path in ("tf32", "tf32x3"):
            v = np.float32(np.uint32(v | (np.uint32(0x80000000) if sign < 0 else 0)).view(np.float32))
            out_a[r, 30] = v
            if i < len(big):
                out_b[40, 50 + i] = -v
        elif path == "bf16":
            out_a[r, 30] = v | (0x8000 if sign < 0 else 0)
            if i < len(big):
                out_b[40, 50 + i] = v ^ (0x8000 if sign > 0 else 0)
        else:
            out_a[r, 30] = sign * v
            if i < len(big):
                out_b[40, 50 + i] = -sign * v
    return out_a, out_b


def tf32_patterns(seed, count, min_exp=1):
    """float32 bit patterns for the preparation tests: random signs / mantissas over every normal exponent from
    min_exp to 254, exact ties (low 13 bits = 0x1000), carries into the exponent, and the band from 0x7F7FF000 to
    FLT_MAX, both signs.  Finite, no subnormals, no zeros."""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 2 ** 23, size=count, dtype=np.uint32)
    u |= rng.integers(min_exp, 255, size=count, dtype=np.uint32) << np.uint32(23)
    ties = (u[: count // 8] & np.uint32(0xFFFFE000)) | np.uint32(0x1000)
    carries = (u[: count // 16] & np.uint32(0xFF800000)) | np.uint32(0x7FF000)   # mantissa rounds up into the exponent
    band = np.arange(0x7F7FF000, 0x7F800000, 0x101, dtype=np.uint32)
    fixed = np.array([0x3FFFF000, 0x3FFFEFFF, 0x7F7FE000, 0x7F7FEFFF, 0x7F7FFFFF], np.uint32)
    fixed = fixed[(fixed >> np.uint32(23)) >= min_exp]
    special = np.concatenate([ties, carries, band, fixed])
    u[: special.size] = special
    u |= rng.integers(0, 2, size=count, dtype=np.uint32) << np.uint32(31)
    return u.view(np.float32)
