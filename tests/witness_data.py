"""Test infrastructure: data on which the witness of every (type, Map, Min | Max) depends on each k-tile, tie rule,
pair order, NaN and identity (mm_kernel_enqueue_witness; tests/witness_naive.py is the result definition).

`case(dtype, map_op, reduce_op, n, k, m, seed)` returns A (n x k) and B (k x m) in the type (bfloat16 as np.uint16
bits).  Operands are small integers in two bands per (reduce, Map): GOOD, from which the winning terms come (few
levels, so that exact ties are everywhere), and BAD, whose terms lose to every GOOD term.  Every row of A and some
columns of B hold GOOD operands only inside a window of k and BAD ones outside; a term is GOOD when both of its
operands are (Add, Multiply, and the Map that can only worsen the term: Max under Min, Min under Max, And under
Max), or when either is (Min under Min, Max under Max, And under Min), and the windows of the columns follow.
Row r's window is, by r % 4: one k-tile (tile r // 4 mod the k-tiles: every k-tile holds winners), a random span,
all of K, or alternately [0, 1) and [K - 1, K) (winners at k = 0 and at k = K - 1).

On top of that:
  * element (ROW_ID, COL_ID): every term equals the reduce's identity (Map(identity, 0 | 1 | identity)): the literal
    rule keeps the last one (W = K - 1), FMNMX none (W = NONE), C is the identity either way;
  * floating types: NaN in B at one or two k of every column j = 3 mod 11 (a NaN term for every literal Map);
  * floating types under Max: row ROW_NONE has every term below the positive identity numeric_limits::min()
    (column COL_NONE too, for the Max Map), so W is NONE there; under Min (not And) its terms are +inf, above
    numeric_limits::max(), with the same effect.  No integer term can be worse than the identity, so integer
    witnesses are never NONE.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import semiring_data as sd  # noqa: E402
from semiring_data import ADD, AND, FLOATING, MAX, MIN, MULTIPLY  # noqa: E402

ROW_ID, COL_ID = 130, 131
ROW_NONE, COL_NONE = 258, 200
NAN_COLS = 11   # columns j with j % NAN_COLS == 3 carry NaN in B

# (GOOD levels, BAD level) of the operands per (reduce, Map); And draws GOOD operands with zeros among them
_LEVELS = {
    (MIN, MULTIPLY): ((1, 2, 3, 4), 20),
    (MIN, ADD): ((1, 2, 3, 4), 12),
    (MIN, MIN): ((1, 2, 3, 4), 12),
    (MIN, MAX): ((1, 2, 3, 4), 12),
    (MIN, AND): ((0, 1, 2), 3),
    (MAX, MULTIPLY): ((5, 6, 7, 8), 1),
    (MAX, ADD): ((8, 9, 10, 11), 1),
    (MAX, MIN): ((8, 9, 10, 11), 1),
    (MAX, MAX): ((8, 9, 10, 11), 1),
    (MAX, AND): ((0, 1, 2), 0),
}
# Maps whose term is GOOD when either operand is: the columns of B are BAD outside their (few) windows
_EITHER = {(MIN, MIN), (MIN, AND), (MAX, MAX)}


def _window(rng, r, k, bk):
    tiles = k // bk
    kind = r % 4
    if kind == 0:
        t = (r // 4) % tiles
        return t * bk, (t + 1) * bk
    if kind == 1:
        lo = int(rng.integers(0, k))
        return lo, int(rng.integers(lo + 1, k + 1))
    if kind == 2:
        return 0, k
    return (0, 1) if (r // 4) % 2 == 0 else (k - 1, k)


def _draw(rng, reduce_op, map_op, shape):
    good, _ = _LEVELS[(reduce_op, map_op)]
    if map_op == AND:   # Min: a zero wins (rare); Max: a nonzero pair wins (zeros common)
        p = (0.15, 0.425, 0.425) if reduce_op == MIN else (0.3, 0.35, 0.35)
        return rng.choice(np.array(good, dtype=np.float64), size=shape, p=p)
    return rng.choice(np.array(good, dtype=np.float64), size=shape)


def case(dtype, map_op, reduce_op, n, k, m, seed):
    """(A n x k, B k x m) in the type, bfloat16 as np.uint16 bits."""
    assert reduce_op in (MIN, MAX)
    rng = np.random.default_rng([seed, dtype, map_op, reduce_op, n, k, m, 7])
    _, bad = _LEVELS[(reduce_op, map_op)]
    bk = sd.bk(dtype)
    either = (reduce_op, map_op) in _EITHER
    a = np.full((n, k), float(bad))
    b = np.full((k, m), float(bad))
    for r in range(n):
        lo, hi = _window(rng, r, k, bk)
        a[r, lo:hi] = _draw(rng, reduce_op, map_op, hi - lo)
    for j in range(m):
        if j % 5 == 0:
            lo, hi = _window(rng, j // 5, k, bk)
        elif either:
            continue                       # BAD everywhere: the row decides
        else:
            lo, hi = 0, k
        b[lo:hi, j] = _draw(rng, reduce_op, map_op, hi - lo)

    if map_op != AND:                      # every term of (ROW_ID, COL_ID) is the identity
        ident = float(sd._Arith(dtype).load(np.array([sd.identity(dtype, reduce_op)]))[0])
        a[ROW_ID, :] = ident
        b[:, COL_ID] = {ADD: 0.0, MULTIPLY: 1.0, MIN: ident, MAX: ident}[map_op]
    if dtype in FLOATING:
        if reduce_op == MAX:               # terms below numeric_limits::min(): W = NONE
            a[ROW_NONE, :] = {MULTIPLY: -1.0, ADD: -1000.0, MIN: -1.0, MAX: -1.0, AND: 0.0}[map_op]
            if map_op == MAX:
                b[:, COL_NONE] = -1.0
        elif map_op != AND:                # Min: +inf terms, worse than numeric_limits::max(): W = NONE
            a[ROW_NONE, :] = np.inf
            if map_op == MIN:
                b[:, COL_NONE] = np.inf
        for j in range(3, m, NAN_COLS):
            b[rng.choice(k, size=1 + j % 2, replace=False), j] = np.nan
    return sd._cast(dtype, a), sd._cast(dtype, b)
