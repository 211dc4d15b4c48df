"""The closure restatement (tests/closure_naive.py) and the data of tests/test_closure_gpu.py, without a GPU.

- On exact data the blocked restatement equals classical sequential Floyd-Warshall for several b, b not dividing N
  included, and its min-plus result equals scipy.sparse.csgraph.floyd_warshall (inf for absent edges).
- The GPU data rejects the plausible wrong closures of closure_naive's `defect` list: each defect changes the result
  on the data the GPU tests use, or a stated reason says why it cannot show there.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closure_data as cd  # noqa: E402
import closure_naive as cn  # noqa: E402
import semiring_data as sd  # noqa: E402
from semiring_data import ADD, AND, FLOAT, INT32, MAX, MIN, MULTIPLY, UINT8  # noqa: E402

# (dtype, map, reduce) whose arithmetic is exact on cd.case(..., exact=False): no rounding, no wrap, no NaN or -0
EXACT_PAIRS = [(INT32, ADD, MIN), (FLOAT, ADD, MIN), (sd.DOUBLE, MIN, MAX), (FLOAT, MAX, MIN), (UINT8, AND, MAX),
               (sd.HALF, MIN, MAX), (sd.UINT32, MAX, MIN), (FLOAT, AND, MAX)]


@pytest.mark.parametrize("b", [8, 16, 24, 48])
@pytest.mark.parametrize("pair", EXACT_PAIRS, ids=[sd.pair_name(*p) for p in EXACT_PAIRS])
def test_blocked_equals_sequential_floyd_warshall(pair, b):
    dt, mp, rd = pair
    n = 40 if dt != UINT8 else 64    # 40 = 5 blocks of 8, 2.5 of 16, 1.7 of 24
    d = cd.case(dt, mp, rd, n, seed=3, exact=False)[0]
    assert sd.same(cn.closure(dt, mp, rd, d, b=b), cn.floyd_warshall(dt, mp, rd, d))


@pytest.mark.parametrize("b", [16, 128])
def test_min_plus_equals_scipy(b):
    csgraph = pytest.importorskip("scipy.sparse.csgraph")
    rng = np.random.default_rng(11)
    n = 272
    w = rng.integers(1, 100, (n, n)).astype(np.float64)
    w[rng.random((n, n)) < 0.9] = np.inf   # absent edges
    np.fill_diagonal(w, 0.0)               # reflexive paths are the caller's to set
    want = csgraph.floyd_warshall(w, directed=True)
    got = cn.closure(sd.DOUBLE, ADD, MIN, w, b=b)
    assert np.array_equal(got, want)
    assert np.isfinite(got).sum() > n      # paths of several hops exist


def test_reliability_keeps_its_zeros():
    """(Multiply, Max): "no path" stays 0; seeding phase 3 with the identity (FLT_MIN) would not."""
    d = np.zeros((256, 256), np.float32)
    d[np.arange(255), np.arange(1, 256)] = 0.5     # a chain: j reachable from i only for j > i
    got = cn.closure(FLOAT, MULTIPLY, MAX, d)
    assert (got[np.tril_indices(256)] == 0).all()
    assert got[0, 3] == np.float32(0.125)
    bad = cn.closure(FLOAT, MULTIPLY, MAX, d, defect="identity_seed")
    assert not sd.same(got, bad)


# the defects and the GPU cases they must change; (reason) where one cannot show
DEFECTS = ["skip_round:0", "skip_round:1", "skip_round:2", "no_panels", "stale_panels", "pivot_rows", "skip_tile",
           "identity_seed", "gauss_seidel", "flavour", "other_problem"]

# defect -> a GPU case (dtype, map, reduce, exact, n, batch) on which it changes D; "dag" = the identity-trap data,
# "nan" = the NaN-term case.  The float Min / Max flavours differ only on NaN terms and on the sign of a zero tie (which
# the FMNMX restatement does not model, so the FMNMX data has no -0): the flavour shows on the NaN-term case.
# An extra evaluation of block row r (pivot_rows) and an in-place step (gauss_seidel) cannot change an idempotent
# closure on data without negative cycles: after phase 2 the row panel already satisfies every relation through K_r,
# and with D[k][k] >= 0 (Add, Min) step k leaves row and column k as they were.  Both show on (Add, Max) int32 data,
# whose positive cycles make every step count (and wrap, identically in the kernel and the restatement).
SHOWN_ON = {
    "skip_round:0": (INT32, ADD, MIN, True, 2 * 128 + 16, 1),
    "skip_round:1": (FLOAT, ADD, MIN, True, 2 * 128 + 16, 1),
    "skip_round:2": (UINT8, AND, MAX, True, 2 * 128 + 64, 1),
    "no_panels": (FLOAT, MIN, MAX, False, 3 * 128, 1),
    "stale_panels": (INT32, ADD, MIN, True, 3 * 128, 1),
    "pivot_rows": (INT32, ADD, MAX, True, 2 * 128 + 16, 1),
    "skip_tile": (sd.DOUBLE, ADD, MIN, True, 3 * 128, 1),
    "identity_seed": (FLOAT, MULTIPLY, MAX, True, 2 * 128 + 16, "dag"),
    "gauss_seidel": (INT32, ADD, MAX, True, 128, 1),
    "flavour": (FLOAT, ADD, MIN, True, 2 * 128 + 16, "nan"),
    "other_problem": (INT32, ADD, MIN, True, 2 * 128 + 16, 3),
}


@pytest.mark.parametrize("defect", DEFECTS)
def test_gpu_data_rejects(defect):
    dt, mp, rd, exact, n, batch = SHOWN_ON[defect]
    if batch == "dag":
        d = cd.reliability_dag(n)
    else:
        d = cd.case(dt, mp, rd, n, seed=5, exact=exact, batch=1 if batch == "nan" else batch, nan_term=batch == "nan")
    fm = dt == FLOAT and not exact
    good = cn.closure(dt, mp, rd, d, fmnmx=fm)
    bad = cn.closure(dt, mp, rd, d, fmnmx=fm, defect=defect)
    assert not sd.same(good, bad), defect


def test_flavour_cannot_show_without_nan_terms():
    """Why the flavour defect is shown on the NaN-term case: on data without NaN terms and without -0, fminf / fmaxf
    and the literal operators give the same bits."""
    d = cd.case(FLOAT, ADD, MIN, 2 * 128 + 16, seed=5, exact=False)
    assert sd.same(cn.closure(FLOAT, ADD, MIN, d, fmnmx=True), cn.closure(FLOAT, ADD, MIN, d, fmnmx=False))


def test_gauss_seidel_cannot_show_on_idempotent_min_plus_with_zero_diagonal():
    """Why the in-place step is shown on data without a reflexive diagonal: with D[k][k] = 0 and (Add, Min) the step
    k leaves row k and column k unchanged, so in-place and simultaneous steps agree."""
    d = cd.case(INT32, ADD, MIN, 128, seed=5, exact=True)[0]
    np.fill_diagonal(d, 0)
    assert sd.same(cn.closure(INT32, ADD, MIN, d), cn.closure(INT32, ADD, MIN, d, defect="gauss_seidel"))
