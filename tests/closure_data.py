"""Test infrastructure: closure inputs (tests/test_closure_gpu.py, tests/test_closure_cpu.py).

`case(dtype, map_op, reduce_op, n, seed, exact, batch)` draws D (batch x N x N) where the best paths cross blocks in
every round: off-cycle entries are drawn from a range of mediocre values and a random Hamiltonian cycle through all N
vertices carries the best value, so the closure of most (i, j) follows the cycle through many blocks.  Under
MM_FLAG_EXACT the floating types also get +0 / -0 entries (ties whose sign shows the operand order) and a NaN at
D[N-1][N-1] (an accumulator that a literal Min / Max replaces by its first term).  At float flags 0 (FMNMX) the data
has no -0 and no NaN, and no operation on it makes one: there fminf / fmaxf give the literal operators' bits.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bf16_naive  # noqa: E402
import semiring_data as sd  # noqa: E402

MIN, MAX, ADD, MULTIPLY, AND = sd.MIN, sd.MAX, sd.ADD, sd.MULTIPLY, sd.AND


def _values(dtype, map_op, reduce_op, rng, shape):
    fl = dtype in sd.FLOATING
    if map_op == ADD:
        lo, hi = (20, 60) if reduce_op == MIN else (1, 20)
        if dtype == sd.UINT8:
            lo, hi = (5, 15) if reduce_op == MIN else (1, 5)
        return rng.integers(lo, hi, shape).astype(np.float64)
    if map_op == MULTIPLY:
        if fl:
            return rng.integers(1, 12, shape) / 16.0 if reduce_op == MAX else rng.integers(17, 40, shape) / 16.0
        return rng.integers(0, 4, shape).astype(np.float64)
    if map_op == AND:
        v = (rng.random(shape) < 0.01).astype(np.float64)
        if fl:
            v[rng.random(shape) < 0.003] = 0.5   # nonzero, not 1
        return v
    hi = 250 if dtype in (sd.UINT8, sd.HALF, sd.BF16) else 1000
    return rng.integers(1, hi, shape).astype(np.float64)


def _best(dtype, map_op, reduce_op):
    if map_op == ADD:
        return 1.0 if reduce_op == MIN else (9.0 if dtype == sd.UINT8 else 30.0)
    if map_op == MULTIPLY:
        return 1.0
    if map_op == AND:
        return 1.0
    return 0.0 if reduce_op == MIN else (255.0 if dtype in (sd.UINT8, sd.HALF, sd.BF16) else 2000.0)


def _cast(dtype, x):
    if dtype == sd.BF16:
        return bf16_naive.from_float(x.astype(np.float32))
    return x.astype(sd.NP[dtype])


def case(dtype, map_op, reduce_op, n, seed, exact=True, batch=1, nan_term=False):
    """nan_term: also a NaN at D[0][N-1], a term from round 0 on: a literal Min / Max keeps it, FMNMX drops it."""
    rng = np.random.default_rng([seed, dtype, map_op, reduce_op, n, batch])
    out = []
    for _ in range(batch):
        d = _values(dtype, map_op, reduce_op, rng, (n, n))
        perm = rng.permutation(n)
        d[perm, np.roll(perm, -1)] = _best(dtype, map_op, reduce_op)
        if exact and dtype in sd.FLOATING:
            z = rng.random((n, n)) < 0.5 / n   # about half a zero per row: ties, not a zero-cost graph
            d[z] = np.where(rng.random(z.sum()) < 0.5, 0.0, -0.0)
            d[n - 1, n - 1] = np.nan
        if nan_term:
            d[0, n - 1] = np.nan
        out.append(_cast(dtype, d))
    return np.stack(out)


def reliability_dag(n):
    """float (Multiply, Max): a chain i -> i + 1 of probability 1/2 plus a few random forward edges; 0 = no edge, and
    every (i, j) with j <= i keeps its 0 in the closure."""
    rng = np.random.default_rng(n)
    d = np.zeros((n, n), np.float32)
    d[np.arange(n - 1), np.arange(1, n)] = 0.5
    i, j = rng.integers(0, n, (2, 4 * n))
    fwd = i < j
    d[i[fwd], j[fwd]] = rng.integers(1, 8, fwd.sum()) / 8.0
    return d
