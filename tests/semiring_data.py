"""Test infrastructure: data on which every CUDA-core semiring kernel's C depends on every k-tile, seed and rounding,
and a numpy restatement of Naive<> that can be told to get one of those wrong.

`discriminating(dtype, map_op, reduce_op, n, k, m, seed, exact)` returns A (n x k) and B (k x m), bfloat16 as np.uint16
bits, drawn for that pair.  The recipe is chosen by the reduce (and the Map when it is And, whose outputs are 0 or 1):

* Product: integers get odd Map outputs (units modulo 2^bits, so C never collapses to 0); floating types get Map
  outputs of magnitude near 1 with random signs and full mantissas, so C stays far from overflow and every factor
  changes its sign or rounding.
* Sum: integers are full range; floating operands are +-m 2^e with e in [-3, 3], so the rounding depends on the order.
  Under `exact`, element (SUM_ZERO, SUM_ZERO) sees only -0 Map outputs: Naive<> gives +0 there, a -0 seed -0.
* Min / Max: levels.  Every row of A has one planted operand at an even k, every column of B one at an odd k, whose
  Map output lies beyond every Map output of two bulk operands; so the extreme of each element sits at one of its two
  plants, and the plants cover every k-tile (row and column PROBE * t: k-tile t) and the last k (column
  PROBE * k-tiles).  Floating types add element (IDENT, IDENT), whose Map outputs are all negative (Max: C is the
  identity numeric_limits::min()) or, under `exact`, all +inf (Min: C is numeric_limits::max()).
* And (as reduce; or And Map under Min / Product): mostly nonzero Map outputs.  At one k in every k-tile, and at the
  last k, some pairs (A[i, k], B[k, j]) give a zero Map output while every other pair stays nonzero.  Under `exact`,
  floating types also get negative operands, -0 outputs at two more k and NaN outputs at a third (nz(NaN) is true).
* And Map under Max: mostly zero Map outputs, nonzero at a few k per element (a boolean product), so both 0 and 1
  appear and C = 0 shows Max's identity for floating types.  Under Sum: a boolean product over every k (counts).

Without `exact` (float Min / Max on the FMNMX kernels) no operand is NaN, -0 or infinite and no Map output is -0.

`simulate(...)` is Naive<> (acc = identity; for k: acc = Reduce(acc, Map(a, b)), one rounding each) in numpy, with the
defects the CPU suite feeds it: skipped k, a wrong seed, other orders of reduction, a contracted Map-Reduce and wrong
nz().  tests/test_semiring_data_cpu.py pins its default against the oracle bit for bit.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bf16_naive  # noqa: E402

HALF, FLOAT, DOUBLE, INT32, UINT32, UINT8, BF16 = range(7)
MULTIPLY, ADD, MIN, MAX, AND = range(5)
TYPES = [HALF, FLOAT, DOUBLE, INT32, UINT32, UINT8, BF16]
OPS = [MULTIPLY, ADD, MIN, MAX, AND]
TYPE_NAME = {HALF: "half", FLOAT: "float", DOUBLE: "double", INT32: "int32", UINT32: "uint32", UINT8: "uint8",
             BF16: "bf16"}
OP_NAME = {MULTIPLY: "mul", ADD: "add", MIN: "min", MAX: "max", AND: "and"}
NP = {HALF: np.float16, FLOAT: np.float32, DOUBLE: np.float64, INT32: np.int32, UINT32: np.uint32, UINT8: np.uint8,
      BF16: np.uint16}
SIZE = {HALF: 2, FLOAT: 4, DOUBLE: 8, INT32: 4, UINT32: 4, UINT8: 1, BF16: 2}
FLOATING = (HALF, FLOAT, DOUBLE, BF16)

TILE = 128          # the C tile of both semiring kernels (rows and columns)
PROBE = 8           # rows and columns 0, 8, 16, ... carry the plants and the special elements
IDENT = PROBE * 12  # Min / Max: the element whose C is the reduce's identity
SUM_ZERO = PROBE * 13   # Sum under exact: the element whose Map outputs are all -0
OK = PROBE * 15      # And: the row of A and column of B whose Map outputs are never zero
TINY = {HALF: 2.0 ** -13, BF16: 2.0 ** -70, FLOAT: 2.0 ** -80, DOUBLE: 2.0 ** -600}   # TINY * TINY rounds to 0


def bk(dtype):
    """Elements of K per k-tile: 64 bytes (the memory width)."""
    return 64 // SIZE[dtype]


def gpu_shape(dtype):
    """N = 259 (three row tiles, the last of 3 rows), M = 256 + w (three column tiles, the last partial), K = 10 k-tiles."""
    return 259, 256 + bk(dtype), 10 * bk(dtype)


def probes(n, m):
    return np.r_[np.arange(0, n, PROBE), n - 1], np.r_[np.arange(0, m, PROBE), m - 1]


def pair_name(dtype, map_op, reduce_op):
    return "%s-%s-%s" % (TYPE_NAME[dtype], OP_NAME[map_op], OP_NAME[reduce_op])


# ---- the data ----------------------------------------------------------------------------------------------------

def _cast(dtype, x):
    """float64 / int64 values -> the type (integers wrap, floating types round to nearest); bfloat16 as bits."""
    if dtype == BF16:
        return bf16_naive.from_double(x)
    if dtype in FLOATING:
        return np.asarray(x, dtype=np.float64).astype(NP[dtype])
    return np.asarray(x).astype(np.int64).astype(NP[dtype])


def _tile_positions(rng, k, b):
    """One k in each k-tile, and the last k."""
    return sorted(set([t * b + int(rng.integers(0, b)) for t in range(k // b)] + [k - 1]))


def _signs(rng, shape):
    return rng.choice(np.array([-1.0, 1.0]), size=shape)


def _odd(rng, dtype, shape):
    lo, hi = {INT32: (-2 ** 30, 2 ** 30), UINT32: (0, 2 ** 31), UINT8: (0, 128)}[dtype]
    return rng.integers(lo, hi, size=shape, dtype=np.int64) * 2 + 1


def _product(dtype, map_op, rng, n, k, m):
    if dtype not in FLOATING:
        a = _odd(rng, dtype, (n, k))
        b = _odd(rng, dtype, (k, m))
        if map_op == ADD:
            b = b - 1           # odd + even is odd
        elif map_op == MULTIPLY:
            # C = (prod_k a_ik) (prod_k b_kj): no two adjacent columns may share the product of B's column
            mod = 2 ** (8 * SIZE[dtype])
            col = [1] * m
            for j in range(m):
                for x in b[:, j]:
                    col[j] = col[j] * int(x) % mod
                if j and col[j] == col[j - 1]:
                    b[0, j] += 2
                    col[j] = col[j] * pow(int(b[0, j]) - 2, -1, mod) * int(b[0, j]) % mod
        return a, b
    near1 = lambda shape: 1.0 + rng.uniform(-1.0 / 16, 1.0 / 16, shape)  # noqa: E731
    a = _signs(rng, (n, k)) * near1((n, k))
    if map_op == ADD:
        return a, rng.uniform(-1.0 / 16, 1.0 / 16, (k, m))
    return a, _signs(rng, (k, m)) * near1((k, m))


def _sum(dtype, map_op, rng, n, k, m, exact):
    if dtype not in FLOATING:
        lo, hi = {INT32: (-2 ** 31, 2 ** 31), UINT32: (0, 2 ** 32), UINT8: (0, 256)}[dtype]
        a, b = rng.integers(lo, hi, size=(n, k), dtype=np.int64), rng.integers(lo, hi, size=(k, m), dtype=np.int64)
        if map_op == ADD:   # C = sum_k a_ik + sum_k b_kj: no two adjacent columns may share B's column sum
            col = b.sum(axis=0) % 2 ** (8 * SIZE[dtype])
            for j in range(1, m):
                if col[j] == col[j - 1]:
                    b[0, j] += 1
                    col[j] += 1
        return a, b
    spread = lambda shape: _signs(rng, shape) * rng.uniform(1, 2, shape) * np.exp2(rng.integers(-3, 4, shape))  # noqa
    a, b = spread((n, k)), spread((k, m))
    if exact:
        a[SUM_ZERO, :] = -0.0
        b[:, SUM_ZERO] = np.abs(b[:, SUM_ZERO]) if map_op == MULTIPLY else -0.0
    return a, b


# (bulk, extreme) operand bands [lo, hi) of the level recipe, per (reduce, Map); "const": the value every column
# (row) of B (A) takes at another row's (column's) plant, so that Map(plant, const) = plant
_LEVELS = {
    (MIN, MULTIPLY): ((8, 16), (1, 4), None),
    (MIN, ADD): ((96, 128), (0, 32), None),
    (MIN, MIN): ((128, 256), (0, 128), None),
    (MIN, MAX): ((128, 256), (0, 32), 0),
    (MAX, MULTIPLY): ((1, 5), (50, 64), None),
    (MAX, ADD): ((0, 32), (96, 128), None),
    (MAX, MAX): ((0, 128), (128, 256), None),
    (MAX, MIN): ((0, 128), (128, 255), 255),
}


def _apart(v, lo, hi):
    """v with no two neighbours in the same integer level: adjacent rows and columns of C then differ."""
    v = v.copy()
    for j in range(1, len(v)):
        if np.floor(v[j]) == np.floor(v[j - 1]):
            v[j] = lo + (np.floor(v[j]) - lo + 1) % (hi - lo) + (v[j] - np.floor(v[j]))
    return v


def _extremes(dtype, map_op, reduce_op, rng, n, k, m, exact):
    (b0, b1), (e0, e1), const = _LEVELS[(reduce_op, map_op)]
    fl = dtype in FLOATING

    def draw(lo, hi, shape):
        if fl:   # a fraction in [0, 1/2): bfloat16 keeps the bands apart after rounding
            return rng.integers(lo, hi, size=shape) + rng.uniform(0, 0.5, shape)
        return rng.integers(lo, hi, size=shape).astype(np.float64)

    a, b = draw(b0, b1, (n, k)), draw(b0, b1, (k, m))
    tiles = k // bk(dtype)
    evens, odds = np.arange(0, k, 2), np.arange(1, k, 2)
    p = rng.choice(evens, size=n)               # row i's plant at k = p[i]
    q = rng.choice(odds, size=m)                # column j's plant at k = q[j]
    for t in range(tiles):                      # rows / columns PROBE * t: a plant in k-tile t
        p[PROBE * t] = t * bk(dtype) + 2 * int(rng.integers(0, bk(dtype) // 2))
        q[PROBE * t] = t * bk(dtype) + 1 + 2 * int(rng.integers(0, bk(dtype) // 2))
    q[PROBE * tiles] = k - 1
    if const is not None:
        b[np.unique(p), :] = const
        a[:, np.unique(q)] = const
    a[np.arange(n), p] = _apart(draw(e0, e1, n), e0, e1)
    b[q, np.arange(m)] = _apart(draw(e0, e1, m), e0, e1)
    if fl and reduce_op == MAX:                 # every Map output below numeric_limits::min()
        a[IDENT, :] = {MULTIPLY: -1.5, ADD: -1000.0, MIN: -1.0, MAX: -1.0}[map_op]
        if map_op == MAX:
            b[:, IDENT] = -1.0
    if fl and reduce_op == MIN and exact:       # every Map output +inf
        a[IDENT, :] = np.inf
        if map_op == MIN:
            b[:, IDENT] = np.inf
    return a, b


# zeroing pairs of the And recipe per Map: (Za, Sa, Zb, Sb) with Map(Za, Zb) == 0 and Map(Za, Sb), Map(Sa, Zb),
# Map(Sa, Sb) nonzero; None: a zero operand zeroes every output (then A and B take turns)
def _zero_pairs(dtype, map_op, negzero):
    fl = dtype in FLOATING
    z = -0.0 if negzero else 0.0
    if map_op == MULTIPLY:
        if fl:
            return (TINY[dtype], 1.0, TINY[dtype], 1.0) if not negzero else (TINY[dtype], 1.0, -TINY[dtype], 1.0)
        shift = 4 if dtype == UINT8 else 16       # 2^shift * odd times 2^shift * odd wraps to 0
        return (2 ** shift * 3, 3, 2 ** shift * 5, 5)
    if map_op == ADD:
        return (z, 1.0, z, 1.0) if negzero else (3.0, 1.0, -3.0, 1.0)
    if map_op == MIN:
        if dtype in (UINT32, UINT8):
            return None
        return (z, 1.0, 2.0, -1.0)
    if map_op == MAX:
        return (z, 1.0, z, 1.0)
    return None                                 # And


def _plant(rng, a, b, kk, pairs, z, side, pa, pb):
    """Zero some Map outputs at k = kk: pairs (Za, Sa, Zb, Sb), or (outer) zeros in A's column (side 0) or B's row."""
    n, m = a.shape[0], b.shape[1]
    if pairs is None:
        a[:, kk] = np.where(rng.random(n) < pa, z, 1.0) if side == 0 else 1.0
        b[kk, :] = np.where(rng.random(m) < pb, z, 1.0) if side == 1 else 1.0
    else:
        za, sa, zb, sb = pairs
        a[:, kk] = np.where(rng.random(n) < pa, za, sa)
        b[kk, :] = np.where(rng.random(m) < pb, zb, sb)


def _nonzero(dtype, map_op, rng, shape, side, exact):
    """Operands whose Map outputs are never zero: odd integers (odd + even for Add); floating |a| in [1, 2),
    |b| in [1/8, 1/2) so that a + b cannot cancel, random signs."""
    if dtype not in FLOATING:
        x = _odd(rng, dtype, shape)
        return x - 1 if (map_op == ADD and side == "b") else x
    mag = rng.uniform(1, 2, shape) if side == "a" else rng.uniform(0.125, 0.5, shape)
    return _signs(rng, shape) * mag if (exact or map_op != MULTIPLY) else mag


def _and_like(dtype, map_op, rng, n, k, m, exact):
    a = _nonzero(dtype, map_op, rng, (n, k), "a", exact)
    b = _nonzero(dtype, map_op, rng, (k, m), "b", exact)
    w = bk(dtype)
    picks = [t * w + rng.choice(w, size=3, replace=False) for t in range(k // w)]
    cover = sorted(set([int(p[0]) for p in picks] + [k - 1]))
    rest = [int(x) for p in picks for x in p[1:] if int(x) != k - 1]
    rng.shuffle(rest)
    special = exact and dtype in FLOATING
    slots = [(kk, False) for kk in cover] + [(kk, True) for kk in (rest[:2] if special else [])]
    plain = rest[3:] if special else rest
    outer = _zero_pairs(dtype, map_op, False) is None
    pa, pb = (0.05, 0.05) if outer else (0.25, 0.1)
    for i, (kk, neg) in enumerate(slots + [(kk, False) for kk in plain]):
        _plant(rng, a, b, kk, _zero_pairs(dtype, map_op, neg), -0.0 if neg else 0.0, i % 2, pa, pb)
    sa, sb = (1.0, 1.0) if outer else _zero_pairs(dtype, map_op, False)[1::2]
    if not outer:   # every column meets a zero at a k of its own, so that adjacent columns of C differ
        zb = _zero_pairs(dtype, map_op, False)[2]
        for j in range(m):
            if j != OK and not (j % PROBE == 0 and j // PROBE < len(slots)):
                b[plain[j % len(plain)], j] = zb
                if j and np.array_equal(b[plain, j] == zb, b[plain, j - 1] == zb):   # flip one more k
                    kk = plain[(j + len(plain) // 2) % len(plain)]
                    b[kk, j] = sb if b[kk, j] == zb else zb
    if special:                                 # NaN Map outputs, which nz() counts as nonzero
        a[:, rest[2]] = 1.0
        b[rest[2], :] = np.where(rng.random(m) < 0.3, np.nan, 1.0)
    planted = [kk for kk, _ in slots] + plain
    # row and column OK see no zero; element (PROBE i, OK) (outer, even i), (OK, PROBE i) (outer, odd i) or
    # (PROBE i, PROBE i) sees exactly one, at slot i
    a[OK, planted], b[planted, OK] = sa, sb
    for i, (kk, neg) in enumerate(slots):
        r = c = PROBE * i
        a[r, planted], b[planted, c] = sa, sb
        pairs = _zero_pairs(dtype, map_op, neg)
        z = -0.0 if neg else 0.0
        if pairs is None:
            if i % 2 == 0:
                a[r, kk] = z
            else:
                b[kk, c] = z
        else:
            a[r, kk], b[kk, c] = pairs[0], pairs[2]
    if outer:   # C's rows and columns take two values: row / column j < 3 of tile t is zeroed iff j == t
        for t in range(3):
            for j in range(3):
                idx = TILE * t + j
                if idx < n:
                    a[idx, planted] = 1.0
                    if j == t:
                        a[idx, slots[0][0]] = 0.0
                if idx < m:
                    b[planted, idx] = 1.0
                    if j == t:
                        b[slots[1][0], idx] = 0.0
    return a, b


def _boolean(dtype, rng, n, k, m, exact, ks, pa, pb):
    """And Map data: A and B nonzero with probability pa / pb at the k in ks, and (A) 1 / (B) 0 elsewhere."""
    fl = dtype in FLOATING
    special = exact and fl

    def values(shape, p):
        v = _nonzero(dtype, MULTIPLY, rng, shape, "a", special)
        if special:
            v = np.where(rng.random(shape) < 0.1, np.nan, v)
        zero = np.where(rng.random(shape) < 0.5, -0.0, 0.0) if special else 0.0
        return np.where(rng.random(shape) < p, v, zero)

    a = np.ones((n, k))
    b = np.zeros((k, m))
    a[:, ks] = values((n, len(ks)), pa)
    b[ks, :] = values((len(ks), m), pb)
    return a, b


def discriminating(dtype, map_op, reduce_op, n, k, m, seed, exact=True):
    """(A n x k, B k x m) in the type (bfloat16 as np.uint16 bits) on which C depends on every k-tile of the pair."""
    rng = np.random.default_rng([seed, dtype, map_op, reduce_op, n, k, m, int(exact)])
    if map_op == AND and reduce_op == MAX:
        ks = sorted(set(_tile_positions(rng, k, bk(dtype)) + list(rng.choice(k, size=30, replace=False))))
        a, b = _boolean(dtype, rng, n, k, m, exact, ks, 0.3, 0.1)
    elif map_op == AND and reduce_op == ADD:
        a, b = _boolean(dtype, rng, n, k, m, exact, list(range(k)), 0.5, 0.5)
    elif reduce_op == AND or map_op == AND:
        a, b = _and_like(dtype, map_op, rng, n, k, m, exact)
    elif reduce_op == MULTIPLY:
        a, b = _product(dtype, map_op, rng, n, k, m)
    elif reduce_op == ADD:
        a, b = _sum(dtype, map_op, rng, n, k, m, exact)
    else:
        a, b = _extremes(dtype, map_op, reduce_op, rng, n, k, m, exact)
    return _cast(dtype, a), _cast(dtype, b)


# ---- Naive<> in numpy, and its defects ---------------------------------------------------------------------------

def identity(dtype, reduce_op):
    """Reduce::identity() in the type (bfloat16 bits)."""
    if dtype == BF16:
        return np.uint16(bf16_naive.IDENTITY[reduce_op])
    t = NP[dtype]
    if reduce_op in (MULTIPLY, AND):
        return t(1)
    if reduce_op == ADD:
        return t(0)
    info = np.finfo(t) if dtype in FLOATING else np.iinfo(t)
    if reduce_op == MIN:
        return t(info.max)
    return t(info.tiny) if dtype in FLOATING else t(info.min)   # Max: numeric_limits<T>::min()


def wrong_seed(dtype, reduce_op):
    """The seed a plausible wrong kernel uses: -0 for Sum, -inf / lowest() for Max, +inf / max() for Min, 0 for And
    and Product.  In an integer type -0 is 0 and +-inf are max() / lowest()."""
    fl = dtype in FLOATING
    if reduce_op == ADD:
        v = -0.0
    elif reduce_op == MAX:
        v = -np.inf if fl else float(np.iinfo(NP[dtype]).min)
    elif reduce_op == MIN:
        v = np.inf if fl else float(np.iinfo(NP[dtype]).max)
    else:
        v = 0.0
    if dtype == BF16:
        return bf16_naive.from_double(np.array([v]))[0]
    return NP[dtype](int(v) if not fl else v)


class _Arith:
    """One type's operations: values carried as numpy arrays of the type (float32 for bfloat16, rounded after
    every operation)."""

    def __init__(self, dtype, nz="exact"):
        self.dtype, self.nz_kind = dtype, nz
        self.bf16 = dtype == BF16
        self.one = np.float32(1) if self.bf16 else NP[dtype](1)
        self.zero = np.float32(0) if self.bf16 else NP[dtype](0)

    def load(self, x):
        return bf16_naive.to_float(x) if self.bf16 else np.asarray(x)

    def store(self, x):
        return bf16_naive.from_float(x) if self.bf16 else x

    def rnd(self, x):
        return bf16_naive.to_float(bf16_naive.from_float(x)) if self.bf16 else x

    def nz(self, x):
        if self.nz_kind == "gt0":
            return x > 0
        if self.nz_kind == "bits":
            return x.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[x.dtype.itemsize]) != 0
        if self.nz_kind == "nan_is_zero":
            return (x != 0) & ~np.isnan(x) if x.dtype.kind == "f" else x != 0
        return x != 0

    def apply(self, op, x, y):
        with np.errstate(all="ignore"):
            if op == MULTIPLY:
                r = x * y
            elif op == ADD:
                r = x + y
            elif op == MIN:
                r = np.where(x < y, x, y)
            elif op == MAX:
                r = np.where(y < x, x, y)
            else:
                r = np.where(self.nz(x) & self.nz(y), self.one, self.zero)
        return self.rnd(r)

    def fma(self, acc, x, y):
        """acc + x * y with one rounding (float64 holds the half / bfloat16 product and sum of this data exactly)."""
        wide = acc.astype(np.float64) + x.astype(np.float64) * y.astype(np.float64)
        if self.bf16:
            return bf16_naive.to_float(bf16_naive.from_double(wide))
        return wide.astype(NP[self.dtype])


def simulate(dtype, map_op, reduce_op, a, b, skip=(), seed=None, order="sequential", contract=False, nz="exact"):
    """C (n x m, bfloat16 bits) = Naive<Map, Reduce>(A n x k, B k x m), or one of its defects:
    skip: k whose terms are left out; seed: the accumulator's initial value instead of the identity;
    order: "sequential" (Naive<>), "swapped" (each step's two k reduced in the other order), "split" (even and odd k in
    two accumulators, combined at the end), "pairwise" (acc (+) (t0 (+) t1)); contract: (Multiply, Add) as one fused
    operation; nz: "exact", "gt0", "bits" (-0 counts as nonzero) or "nan_is_zero"."""
    ar = _Arith(dtype, nz)
    av, bv = ar.load(a), ar.load(b)
    k = av.shape[1]
    init = ar.load(np.array([identity(dtype, reduce_op) if seed is None else seed]))[0]
    acc = np.full((av.shape[0], bv.shape[1]), init, dtype=av.dtype)
    term = lambda kk: ar.apply(map_op, av[:, kk:kk + 1], bv[kk:kk + 1, :])  # noqa: E731
    skip = set(skip)
    if order == "sequential":
        for kk in range(k):
            if kk in skip:
                continue
            if contract:
                acc = ar.fma(acc, av[:, kk:kk + 1], bv[kk:kk + 1, :])
            else:
                acc = ar.apply(reduce_op, acc, term(kk))
    elif order == "swapped":
        for kk in range(0, k, 2):
            acc = ar.apply(reduce_op, ar.apply(reduce_op, acc, term(kk + 1)), term(kk))
    elif order == "pairwise":
        for kk in range(0, k, 2):
            acc = ar.apply(reduce_op, acc, ar.apply(reduce_op, term(kk), term(kk + 1)))
    elif order == "split":
        acc2 = acc.copy()
        for kk in range(0, k, 2):
            acc = ar.apply(reduce_op, acc, term(kk))
            acc2 = ar.apply(reduce_op, acc2, term(kk + 1))
        acc = ar.apply(reduce_op, acc, acc2)
    else:
        raise ValueError(order)
    return ar.store(acc)


def same(x, y):
    """Bit equality, except that any NaN equals any NaN (payloads are free)."""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    if x.shape != y.shape:
        return False
    if x.dtype == np.uint16 and y.dtype == np.uint16:   # bfloat16 bits
        return bf16_naive.same_nan_free(x, y)
    if x.dtype.kind == "f":
        nx, ny = np.isnan(x), np.isnan(y)
        w = {2: np.uint16, 4: np.uint32, 8: np.uint64}[x.dtype.itemsize]
        return bool(np.array_equal(nx, ny) and np.array_equal(x[~nx].view(w), y[~ny].view(w)))
    return bool(np.array_equal(x, y))


def reference(oracle, dtype, map_op, reduce_op, a, b, n, k, m):
    """Naive<> of the whole C: the oracle for six types, tests/bf16_naive.py for bfloat16."""
    if dtype == BF16:
        return bf16_naive.naive(map_op, reduce_op, a, b, n, k, m)
    return oracle.naive(dtype, map_op, reduce_op, a, b, n, k, m, threads=8)
