"""Test infrastructure: the result definition of mm_kernel_enqueue_accumulate, restated on the CPU bit for bit.

    C_new = R(C_old, P)

P is what mm_kernel_enqueue_batched stores for the same arguments; R is one application of the reduce of the path that
computed P, in the data type, with C_old as the FIRST operand (include/mm_b200.h):

  Add       float32 / float64: the IEEE sum, rounded to nearest even (numpy's own arithmetic in the type).  half and
            bfloat16: the sum of two 16-bit values is exact in float64, then rounded once to the type.  Integers wrap
            modulo 2^32, uint8_t modulo 256.
  Multiply  the same with the product (exact in float64 for the 16-bit types).
  Min       literal `(c < p) ? c : p`; FMNMX (float without MM_FLAG_EXACT): fminf -- a NaN operand gives the other,
            -0 is below +0.
  Max       literal `(p < c) ? c : p`; FMNMX: fmaxf likewise.
  And       `(c != 0 && p != 0) ? 1 : 0`, NaN counting as nonzero.

Arrays are numpy arrays of the type; bfloat16 as np.uint16 bit patterns.  Arithmetic results may be any NaN where IEEE
gives a NaN (the hardware's canonical NaN is not restated): compare with `same`.
"""
import numpy as np

import bf16_naive
import semiring_data as sd
from semiring_data import ADD, AND, BF16, DOUBLE, FLOAT, FLOATING, HALF, MAX, MIN, MULTIPLY, UINT8

_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view(_UINT[x.dtype.itemsize])


def _value(dtype, x):
    """The values as float64 (floating types) or int64; bfloat16 bits decoded."""
    if dtype == BF16:
        return bf16_naive.to_float(x).astype(np.float64)
    return np.asarray(x).astype(np.float64 if dtype in FLOATING else np.int64)


def _round(dtype, v):
    """float64 / int64 -> the type: one rounding to nearest even, integers wrap."""
    if dtype == BF16:
        return bf16_naive.from_double(v)
    if dtype in (HALF, FLOAT, DOUBLE):
        return v.astype(sd.NP[dtype])    # numpy converts float64 to half / float with one correct rounding
    return (v & {UINT8: 0xFF}.get(dtype, 0xFFFFFFFF)).astype(np.uint32).astype(sd.NP[dtype])


def _fmnmx(c, p, is_min):
    """fminf / fmaxf on float32: a NaN operand gives the other one, -0 counts below +0."""
    cn, pn = np.isnan(c), np.isnan(p)
    neg_c, neg_p = np.signbit(c), np.signbit(p)
    with np.errstate(invalid="ignore"):
        if is_min:
            pick_c = (c < p) | ((c == p) & neg_c)
        else:
            pick_c = (p < c) | ((c == p) & ~neg_c)
    r = np.where(pick_c, c, p)
    r = np.where(pn & ~cn, c, r)
    return np.where(cn, p, r).astype(np.float32)


def reduce_once(dtype, reduce_op, c, p, fmnmx=False):
    """R(c, p) elementwise, in the type (bfloat16 bits).  fmnmx: the float default Min / Max."""
    c, p = np.asarray(c), np.asarray(p)
    if reduce_op in (MIN, MAX):
        if fmnmx:
            assert dtype == FLOAT
            return _fmnmx(c, p, reduce_op == MIN)
        cv, pv = _value(dtype, c), _value(dtype, p)
        with np.errstate(invalid="ignore"):
            pick_c = (cv < pv) if reduce_op == MIN else (pv < cv)
        return np.where(pick_c, c, p)          # one operand's bits, NaN payloads and signed zeros included
    if reduce_op == AND:
        cv, pv = _value(dtype, c), _value(dtype, p)
        one = (cv != 0) & (pv != 0)            # NaN != 0
        return _round(dtype, one.astype(np.float64 if dtype in FLOATING else np.int64))
    with np.errstate(all="ignore"):
        if dtype in (FLOAT, DOUBLE):           # IEEE arithmetic in the type itself
            return (c + p) if reduce_op == ADD else (c * p)
        cv, pv = _value(dtype, c), _value(dtype, p)
        return _round(dtype, (cv + pv) if reduce_op == ADD else (cv * pv))


def same(dtype, x, y, reduce_op=ADD):
    """Byte equality.  For Add and Multiply on floating types any NaN equals any NaN (an arithmetic NaN's payload is
    the hardware's); Min, Max and And results are one operand's bits or 0 / 1, compared exactly."""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    return x.shape == y.shape and first_difference(dtype, x, y, reduce_op) is None


def first_difference(dtype, x, y, reduce_op=ADD):
    """Index of the first element where `same` fails, or None."""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    bad = _bits(x) != _bits(y)
    if dtype in FLOATING and reduce_op in (ADD, MULTIPLY):
        nan = (lambda b: (b & 0x7FFF) > 0x7F80) if dtype == BF16 else np.isnan
        bad &= ~(nan(x) & nan(y))
    idx = np.argwhere(bad)
    return None if len(idx) == 0 else tuple(int(v) for v in idx[0])


# ---- A and B -----------------------------------------------------------------------------------------------------

# (x, y) with Map(x, y) = +0 and = -0 for each Map (And has no -0 output)
_ZERO_PLANT = {ADD: ((1.0, -1.0), (-0.0, -0.0)), MULTIPLY: ((0.0, 1.0), (-0.0, 1.0)), MIN: ((0.0, 0.0), (-0.0, -0.0)),
               MAX: ((0.0, 0.0), (-0.0, -0.0)), AND: ((0.0, 0.0), (0.0, 0.0))}


def data(dtype, map_op, reduce_op, n, k, m, seed, exact=True):
    """(A n x k, B k x m): semiring_data.discriminating, plus, for a floating Min / Max, products whose P tells the
    literal Min / Max from FMNMX once C_old is reduced into it (the two differ only at a +0 / -0 tie and at a NaN P):
      - rows 1, 130, n - 2 and columns 3, 131, m - 2: every term of those elements of C is +0, so P = +0;
      - under MM_FLAG_EXACT, rows 5, 134, n - 1 and columns 7, 135, m - 4: every term -0, so P = -0;
      - under MM_FLAG_EXACT (Map other than And), columns 9, 137, m - 6 of B's last row are NaN: the last term of those
        columns is NaN, which the literal Min / Max keeps, so P = NaN.
    The float default data stays NaN-free and gets no -0 (there FMNMX and the literal Naive<> agree)."""
    a, b = sd.discriminating(dtype, map_op, reduce_op, n, k, m, seed, exact=exact)
    if dtype not in FLOATING or reduce_op not in (MIN, MAX):
        return a, b
    a, b = a.copy(), b.copy()
    plants = [(_ZERO_PLANT[map_op][0], [1, 130, n - 2], [3, 131, m - 2])]
    if exact:
        plants.append((_ZERO_PLANT[map_op][1], [5, 134, n - 1], [7, 135, m - 4]))
    for (x, y), rows, cols in plants:
        a[rows, :] = _round(dtype, np.array([x]))[0]
        b[:, cols] = _round(dtype, np.array([y]))[0]
    if exact and map_op != AND:
        b[k - 1, [9, 137, m - 6]] = _round(dtype, np.array([np.nan]))[0]
    return a, b


# ---- C_old ------------------------------------------------------------------------------------------------------

def _specials(dtype, reduce_op):
    """The values C_old must contain: NaN, +-0, +-inf (floating types), the identities, the extremes."""
    if dtype in FLOATING:
        vals = [np.nan, 0.0, -0.0, np.inf, -np.inf, 1.0, -1.0]
        out = list(_round(dtype, np.array(vals, dtype=np.float64)))
    else:
        info = np.iinfo(sd.NP[dtype])
        out = [sd.NP[dtype](v) for v in (0, 1, info.max, info.min)]
    return out + [sd.identity(dtype, r) for r in (MULTIPLY, ADD, MIN, MAX, AND)]


def c_old(dtype, reduce_op, p, seed):
    """C_old for an accumulate test whose plain product is p (any shape, in the type): random values of p's magnitude
    everywhere, then on a sparse random sixth of the elements the specials of _specials, on another sixth p itself
    (ties: R(p, p)), and on another sixth p with its sign flipped; where p is +-0, the other zero on half of the
    elements (the tie of +0 and -0).  For And, half of the random values are zero."""
    rng = np.random.default_rng([seed, dtype, reduce_op] + list(p.shape))
    shape = p.shape
    if dtype in FLOATING:
        pv = _value(dtype, p)
        finite = pv[np.isfinite(pv)]
        scale = float(np.abs(finite).max()) if finite.size else 1.0
        scale = scale if scale > 0 else 1.0
        v = rng.uniform(-1.0, 1.0, size=shape) * scale
        c = _round(dtype, v)
    else:
        info = np.iinfo(sd.NP[dtype])
        c = rng.integers(int(info.min), int(info.max) + 1, size=shape, dtype=np.int64).astype(sd.NP[dtype])
    if reduce_op == AND:   # And tells C_old from P only where C_old is zero and P is not
        c = np.where(rng.integers(0, 2, size=shape) == 0, np.zeros(1, dtype=c.dtype), c)
    which = rng.integers(0, 6, size=shape)
    sp = np.array(_specials(dtype, reduce_op), dtype=c.dtype)
    c = np.where(which == 1, sp[rng.integers(0, len(sp), size=shape)], c)
    c = np.where(which == 2, p, c)
    if dtype in FLOATING:
        neg = (_bits(p) ^ (np.array(1, dtype=_bits(p).dtype) << (8 * p.dtype.itemsize - 1))).view(c.dtype)
        c = np.where(which == 3, neg, c)
        # where P is +-0, mostly the other zero: the tie that tells the literal Min / Max from FMNMX
        c = np.where((_value(dtype, p) == 0) & (which >= 3), neg, c)
    return np.ascontiguousarray(c)
