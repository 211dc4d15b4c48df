"""CPU tests of tests/semiring_data.py: the data of tests/test_semiring_coverage_gpu.py rejects wrong semiring kernels.

For every (type, Map, Reduce) at the GPU file's shape (N = 259, M = 256 + w, K = 10 k-tiles), a numpy restatement of
Naive<> (`semiring_data.simulate`), pinned bit for bit to the oracle's Naive<> (bfloat16: tests/bf16_naive.py), runs
each wrong kernel below on the rows and columns that carry the plants (every PROBE-th, and the last).  An element of
C depends only on its row of A and its column of B, so a difference there is a difference in the GPU file's C.

| defect                                                         | applies to                                        |
|----------------------------------------------------------------|---------------------------------------------------|
| the last k-tile skipped; each single k-tile t skipped          | every pair                                        |
| the last k skipped                                             | every pair                                        |
| a wrong seed: -0 (Sum), -inf / lowest() (Max), +inf / max()    | every pair                                        |
| (Min), 0 (And, Product)                                        |                                                   |
| each step's two k reduced in swapped order; even and odd k in  | every pair                                        |
| two accumulators; acc (+) (t0 (+) t1)                          |                                                   |
| Map and Reduce contracted into one rounding                    | half and bfloat16 (Multiply, Add)                 |
| nz(x) as x > 0, as bits != 0 (-0 nonzero), NaN counted as zero | every pair with And as Map or Reduce              |

Each wrong kernel must change at least one element, except where EXEMPT says it cannot, and there it must change
none: the list is checked in both directions.  The whole C (from the oracle) must also have three properties that keep
a swap of tiles or of the packed half2 / bfloat162 lanes visible: no two row tiles equal, no two column tiles equal,
no two adjacent columns equal (with the exemption below).  The FMNMX data (float Min / Max without MM_FLAG_EXACT)
holds no NaN, -0 or infinite operand and no -0 Map output, and rejects the skips and the Max seed.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import semiring_data as sd  # noqa: E402
from semiring_data import ADD, AND, BF16, FLOATING, HALF, INT32, MAX, MIN, MULTIPLY, UINT32, UINT8  # noqa: E402

PAIRS = [(dt, mp, rd) for dt in sd.TYPES for mp in sd.OPS for rd in sd.OPS]
FMNMX = [(sd.FLOAT, mp, rd) for mp in sd.OPS for rd in sd.OPS if {mp, rd} & {MIN, MAX}]
ORDERS = ("swapped", "split", "pairwise")
NZ = ("gt0", "bits", "nan_is_zero")
SEED = 5   # the seed of tests/test_semiring_coverage_gpu.py


def defects(dt, mp, rd):
    tiles = sd.gpu_shape(dt)[2] // sd.bk(dt)
    names = ["skip_tile_%d" % t for t in range(tiles)] + ["skip_last_tile", "skip_last_k", "seed"] + list(ORDERS)
    if dt in (HALF, BF16) and (mp, rd) == (MULTIPLY, ADD):
        names.append("contract")
    if AND in (mp, rd):
        names += ["nz_" + v for v in NZ]
    return names


# Where a defect cannot be observed: (predicate on (type, Map, Reduce, exact), defects, reason)
EXEMPT = [
    (lambda dt, mp, rd, ex: dt not in FLOATING and rd == ADD, ("seed",),
     "an integer type has no -0: the Sum seed is the identity 0"),
    (lambda dt, mp, rd, ex: dt not in FLOATING and rd == MIN, ("seed",),
     "an integer Min seed +inf is max(), the identity, so nothing comes out below it"),
    (lambda dt, mp, rd, ex: dt not in FLOATING and rd == MAX, ("seed",),
     "an integer Max seed lowest() is min(), the identity"),
    (lambda dt, mp, rd, ex: dt in FLOATING and mp == AND and rd == MIN, ("seed",),
     "And outputs are 0 or 1, below Min's identity max() and +inf alike"),
    (lambda dt, mp, rd, ex: dt in FLOATING and mp == AND and rd == ADD, ("seed",),
     "And outputs are +0 or 1, never -0, so a -0 seed is absorbed"),
    (lambda dt, mp, rd, ex: not ex and rd == MIN, ("seed",),
     "the FMNMX data is finite: no element reduces only +inf"),
    (lambda dt, mp, rd, ex: not ex and rd == ADD, ("seed",),
     "the FMNMX data has no -0: no element sums only -0"),
    (lambda dt, mp, rd, ex: rd in (MIN, MAX, AND), ORDERS,
     "Min, Max and And select or test: the order of reduction does not change the result"),
    (lambda dt, mp, rd, ex: dt not in FLOATING, ORDERS,
     "integer + and * are exact modulo 2^bits in any order"),
    (lambda dt, mp, rd, ex: mp == AND, ORDERS,
     "And outputs are 0 or 1: the partial sums are small integers and the partial products 0 or 1, exact in any order"),
    (lambda dt, mp, rd, ex: dt in (UINT32, UINT8), tuple("nz_" + v for v in NZ),
     "unsigned integers: x > 0, bits != 0 and x != 0 agree, and there is no NaN"),
    (lambda dt, mp, rd, ex: dt == INT32, ("nz_bits", "nz_nan_is_zero"),
     "int32 has one zero and no NaN"),
]

# C[i, j] = rowOK[i] and colOK[j] whenever a zero operand zeroes every Map output it meets, so columns take two values
OUTER = lambda dt, mp, rd: (mp == AND and rd in (AND, MIN, MULTIPLY)) or (  # noqa: E731
    mp == MIN and rd == AND and dt in (UINT32, UINT8))


def exemption(dt, mp, rd, exact, defect):
    for pred, names, reason in EXEMPT:
        if defect in names and pred(dt, mp, rd, exact):
            return reason
    return None


_DATA = {}


def data(oracle, dt, mp, rd, exact=True):
    key = (dt, mp, rd, exact)
    if key not in _DATA:
        n, m, k = sd.gpu_shape(dt)
        a, b = sd.discriminating(dt, mp, rd, n, k, m, SEED, exact)
        _DATA[key] = (a, b, sd.reference(oracle, dt, mp, rd, a, b, n, k, m))
    return _DATA[key]


def run_defect(dt, mp, rd, a, b, defect):
    k, bk = a.shape[1], sd.bk(dt)
    kw = {}
    if defect.startswith("skip_tile_"):
        t = int(defect.rsplit("_", 1)[1])
        kw["skip"] = range(t * bk, (t + 1) * bk)
    elif defect == "skip_last_tile":
        kw["skip"] = range(k - bk, k)
    elif defect == "skip_last_k":
        kw["skip"] = (k - 1,)
    elif defect == "seed":
        kw["seed"] = sd.wrong_seed(dt, rd)
    elif defect in ORDERS:
        kw["order"] = defect
    elif defect == "contract":
        kw["contract"] = True
    else:
        kw["nz"] = defect[3:]
    return sd.simulate(dt, mp, rd, a, b, **kw)


def check_rejections(oracle, dt, mp, rd, exact, names):
    a, b, c = data(oracle, dt, mp, rd, exact)
    rows, cols = sd.probes(*c.shape)
    ap, bp = a[rows], b[:, cols]
    right = sd.simulate(dt, mp, rd, ap, bp)
    assert sd.same(right, c[np.ix_(rows, cols)]), "the numpy Naive<> differs from the oracle"
    wrong = []
    for d in names:
        rejected = not sd.same(run_defect(dt, mp, rd, ap, bp, d), right)
        reason = exemption(dt, mp, rd, exact, d)
        if rejected == (reason is not None):
            wrong.append("%s: %s" % (d, ("rejected although exempt (%s)" % reason) if reason else "not rejected"))
    assert not wrong, "; ".join(wrong)


@pytest.mark.parametrize("dt,mp,rd", PAIRS, ids=[sd.pair_name(*p) for p in PAIRS])
def test_data_rejects_wrong_kernels(oracle, dt, mp, rd):
    check_rejections(oracle, dt, mp, rd, True, defects(dt, mp, rd))


@pytest.mark.parametrize("dt,mp,rd", FMNMX, ids=[sd.pair_name(*p) for p in FMNMX])
def test_fmnmx_data_rejects_skips_and_seeds(oracle, dt, mp, rd):
    names = [d for d in defects(dt, mp, rd) if d.startswith("skip") or d == "seed"]
    check_rejections(oracle, dt, mp, rd, False, names)


@pytest.mark.parametrize("dt,mp,rd", FMNMX, ids=[sd.pair_name(*p) for p in FMNMX])
def test_fmnmx_data_stays_inside_the_documented_equality(dt, mp, rd):
    """No NaN, -0 or infinite operand, and no Map output -0 or NaN: there FMNMX equals `(a < b) ? a : b`."""
    n, m, k = sd.gpu_shape(dt)
    a, b = sd.discriminating(dt, mp, rd, n, k, m, SEED, exact=False)
    for x in (a, b):
        assert np.all(np.isfinite(x)) and not np.any((x == 0) & np.signbit(x))
    for kk in range(k):
        t = sd._Arith(dt).apply(mp, a[:, kk:kk + 1], b[kk:kk + 1, :])
        assert not np.any(np.isnan(t)) and not np.any((t == 0) & np.signbit(t)), "k = %d" % kk


def _equal_slices(c, axis, size):
    """Pairs of distinct tiles (along axis) whose overlapping part is equal."""
    count = c.shape[axis]
    tiles = [(s, min(s + size, count)) for s in range(0, count, size)]
    out = []
    for i in range(len(tiles)):
        for j in range(i + 1, len(tiles)):
            h = min(tiles[i][1] - tiles[i][0], tiles[j][1] - tiles[j][0])
            x = np.take(c, range(tiles[i][0], tiles[i][0] + h), axis=axis)
            y = np.take(c, range(tiles[j][0], tiles[j][0] + h), axis=axis)
            if sd.same(x, y):
                out.append((i, j))
    return out


DATA_SETS = [p + (True,) for p in PAIRS] + [p + (False,) for p in FMNMX]


@pytest.mark.parametrize("dt,mp,rd,exact", DATA_SETS,
                         ids=[sd.pair_name(*p[:3]) + ("" if p[3] else "-fmnmx") for p in DATA_SETS])
def test_c_tells_tiles_and_columns_apart(oracle, dt, mp, rd, exact):
    c = data(oracle, dt, mp, rd, exact)[2]
    assert _equal_slices(c, 0, sd.TILE) == [], "equal row tiles"
    assert _equal_slices(c, 1, sd.TILE) == [], "equal column tiles"
    adjacent = [j for j in range(c.shape[1] - 1) if sd.same(c[:, j], c[:, j + 1])]
    if OUTER(dt, mp, rd):
        assert adjacent, "exempt from distinct adjacent columns, yet they are distinct"
    else:
        assert adjacent == [], "equal adjacent columns %s" % adjacent[:8]


@pytest.mark.parametrize("dt,mp,rd", [(sd.FLOAT, MULTIPLY, MAX), (sd.DOUBLE, ADD, MAX), (HALF, MAX, MAX),
                                      (BF16, AND, MAX), (sd.FLOAT, ADD, MIN), (sd.DOUBLE, MIN, MIN),
                                      (HALF, MULTIPLY, MIN), (BF16, MAX, MIN)])
def test_identities_appear_in_c(oracle, dt, mp, rd):
    """Max's numeric_limits::min() and Min's numeric_limits::max() are elements of C."""
    c = data(oracle, dt, mp, rd)[2]
    u = np.dtype("u%d" % c.itemsize)
    assert np.any(np.ascontiguousarray(c).view(u) == np.array([sd.identity(dt, rd)]).view(u)[0])
