"""Test infrastructure: the result definition the library's exact bfloat16 path is held to.

The reference has no bfloat16, so there is no reference Naive<> to pin against.  This module restates
Naive<Map, Reduce> (acc = Reduce::identity(); for k: acc = Reduce(acc, Map(a, b))) for bfloat16 with one
round-to-nearest-even after every Map and every Reduce.  Each operation is computed in float32 and rounded
once to bfloat16.  For +, * and compare that is the correctly rounded bfloat16 result: float's 24
significand bits are >= 2 * 8 + 2, so the float rounding never changes the final one.  Identities as the
reference's functors: Add 0, Multiply 1, And 1, Min numeric_limits::max() (0x7F7F), Max
numeric_limits::min() (0x0080, the smallest positive normal).  Min / Max are the literal `(a < b) ? a : b`.

bfloat16 values are carried as np.uint16 bit patterns.  tests/test_bf16_cpu.py pins this module against an
independent sequential evaluation in torch-CPU bfloat16.
"""
import numpy as np

MULTIPLY, ADD, MIN, MAX, AND = range(5)
IDENTITY = {MULTIPLY: 0x3F80, ADD: 0x0000, MIN: 0x7F7F, MAX: 0x0080, AND: 0x3F80}
ONE, ZERO = np.float32(1.0), np.float32(0.0)


def to_float(bits):
    """bfloat16 bit patterns -> float32 (exact)."""
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def from_float(x):
    """float32 -> bfloat16 bits, to nearest even; a NaN stays a (quiet) NaN."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    r = (u + np.uint32(0x7FFF) + ((u >> 16) & 1)) >> 16
    return np.where(nan, (u >> 16) | 0x0040, r).astype(np.uint16)


def from_double(d):
    """float64 -> bfloat16 bits, correctly rounded (rounding through float32 could round twice)."""
    d = np.asarray(d, dtype=np.float64)
    with np.errstate(all="ignore"):
        e = np.maximum(np.floor(np.log2(np.abs(d))), -126.0)      # below 2^-126: the subnormal quantum 2^-133
        q = np.exp2(e - 7.0)                                       # one unit in the last place at d's binade
        r = np.rint(d / q) * q                                     # ties to even
    r = np.where(np.isfinite(d) & (d != 0), r, d)
    r = np.where(np.abs(r) > 3.3895313892515355e38, np.copysign(np.inf, d), r)   # past the largest finite value
    return from_float(r.astype(np.float32))                       # exact: r is a bfloat16 value (or inf / NaN / 0)


def _apply(op, x, y):
    """One functor application on float32 arrays holding bfloat16 values; bfloat16 bits out."""
    with np.errstate(all="ignore"):
        if op == MULTIPLY:
            return from_float(x * y)
        if op == ADD:
            return from_float(x + y)
        if op == MIN:
            return from_float(np.where(x < y, x, y))
        if op == MAX:
            return from_float(np.where(y < x, x, y))
        if op == AND:
            return from_float(np.where((x != 0) & (y != 0), ONE, ZERO))
    raise ValueError("unknown operator %r" % op)


def naive(map_op, reduce_op, a, b, n, k, m, transposed_a=False):
    """C (n x m, bfloat16 bits) = A (x) B: A n x k (k x n when transposed_a), B k x m, row-major bit patterns."""
    av = to_float(np.asarray(a).reshape(-1)).reshape((k, n) if transposed_a else (n, k))
    if transposed_a:
        av = av.T
    bv = to_float(np.asarray(b).reshape(-1)).reshape(k, m)
    acc = np.full((n, m), IDENTITY[reduce_op], dtype=np.uint16)
    for kk in range(k):
        t = _apply(map_op, av[:, kk:kk + 1], bv[kk:kk + 1, :])
        acc = _apply(reduce_op, to_float(acc), to_float(t))
    return acc


def fill(oracle, n, k, m, seed=5):
    """The reference's input recipe (A drawn first, then B, U[1, 10] doubles) rounded correctly to bfloat16."""
    a, b = oracle.fill(oracle.DOUBLE, n, k, m, seed)
    return from_double(a), from_double(b)


def same_nan_free(x, y):
    """Bit equality, except that any NaN equals any NaN (payloads are free)."""
    x, y = np.asarray(x, dtype=np.uint16).reshape(-1), np.asarray(y, dtype=np.uint16).reshape(-1)
    nx, ny = (x & 0x7FFF) > 0x7F80, (y & 0x7FFF) > 0x7F80
    return bool(np.array_equal(nx, ny) and np.array_equal(x[~nx], y[~ny]))
