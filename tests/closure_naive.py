"""Test infrastructure: the result definition mm_kernel_enqueue_closure is held to (include/mm_b200.h), in numpy.

`closure(dtype, map_op, reduce_op, d, b)` rewrites a copy of D (N x N, or batch x N x N) by blocked Floyd-Warshall
with blocks K_r = [r*b, min((r+1)*b, N)).  A step k updates its (i, j) simultaneously (vectorised: every read sees
the values from before the step), D'[i][j] = R(D[i][j], Map(D[i][k], D[k][j])), one rounding per Map and per Reduce
(float16 through numpy, bfloat16 with the rounding of bf16_naive, integers wrapping like the device).  Round r:
  1. for k in K_r: step k over K_r x K_r;
  2. for k in K_r: step k over K_r x (not K_r) and (not K_r) x K_r;
  3. for (not K_r) x (not K_r): acc = D[i][j]; for k in K_r: acc = R(acc, Map(D[i][k], D[k][j])); D[i][j] = acc.
`fmnmx`: float at flags 0, where Min / Max (as Map and as Reduce) are fminf / fmaxf.

`defect` switches on the wrong closures tests/test_closure_cpu.py shows the GPU data rejects:
  "skip_round:<r>"  round r left out;          "no_panels"      phase 2 left out;
  "stale_panels"    phase 3 reads the panels from before phase 2;
  "pivot_rows"      phase 3 also updates block row r (from the panels as phase 2 left them);
  "skip_tile"       phase 3 leaves the tile of block row r+1 / block column r+2 (mod blocks) as it was;
  "identity_seed"   phase 3 seeds with the reduce's identity and reduces D[i][j] in last;
  "gauss_seidel"    phases 1 and 2 update in place, row by row, reading values already updated in the step;
  "flavour"         the other float Min / Max (literal for FMNMX and the reverse);
  "other_problem"   problem p reads its phase-3 seed from problem (p + 1) % batch.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import semiring_data as sd  # noqa: E402

MIN, MAX, ADD, MULTIPLY, AND = sd.MIN, sd.MAX, sd.ADD, sd.MULTIPLY, sd.AND
B = 128   # mm_closure_block() of every type


class _Ops:
    def __init__(self, dtype, map_op, reduce_op, fmnmx):
        self.ar = sd._Arith(dtype)
        self.map_op, self.reduce_op, self.fmnmx = map_op, reduce_op, fmnmx

    def _op(self, op, x, y):
        if self.fmnmx and op in (MIN, MAX):
            with np.errstate(all="ignore"):
                return (np.fmin if op == MIN else np.fmax)(x, y)
        return self.ar.apply(op, x, y)

    def term(self, x, y):
        return self._op(self.map_op, x, y)

    def red(self, acc, t):
        return self._op(self.reduce_op, acc, t)


def _step(o, d, k, rows, cols, gauss_seidel=False):
    """Step k over rows x cols of d (2-D, values as loaded), in place."""
    if not gauss_seidel:
        d[np.ix_(rows, cols)] = o.red(d[np.ix_(rows, cols)], o.term(d[rows, k][:, None], d[k, cols][None, :]))
        return
    for i in rows:   # in place: a row read after it was updated in this step sees the new values
        d[i, cols] = o.red(d[i, cols], o.term(d[i, k], d[k, cols]))


def _one(o, d, b, defect, seed_from=None):
    n = d.shape[0]
    gs = defect == "gauss_seidel"
    blocks = (n + b - 1) // b
    for r in range(blocks):
        if defect == "skip_round:%d" % r:
            continue
        kr = np.arange(r * b, min((r + 1) * b, n))
        rest = np.setdiff1d(np.arange(n), kr)
        before = d.copy()
        for k in kr:
            _step(o, d, k, kr, kr, gs)
        if defect != "no_panels":
            for k in kr:
                if gs:
                    _step(o, d, k, kr, rest, True)
                    _step(o, d, k, rest, kr, True)
                else:   # the two panels read nothing of each other
                    row = o.red(d[np.ix_(kr, rest)], o.term(d[kr, k][:, None], d[k, rest][None, :]))
                    col = o.red(d[np.ix_(rest, kr)], o.term(d[rest, k][:, None], d[k, kr][None, :]))
                    d[np.ix_(kr, rest)] = row
                    d[np.ix_(rest, kr)] = col
        if len(rest) == 0:
            continue
        src = before if defect == "stale_panels" else d
        rows = np.arange(n) if defect == "pivot_rows" else rest
        cols = rest
        seed_d = seed_from[r] if seed_from is not None else d
        acc = seed_d[np.ix_(rows, cols)].copy()
        if defect == "identity_seed":
            acc = np.full(acc.shape, o.ar.load(np.array([sd.identity(o.ar.dtype, o.reduce_op)]))[0], dtype=acc.dtype)
        for k in kr:
            acc = o.red(acc, o.term(src[rows, k][:, None], src[k, cols][None, :]))
        if defect == "identity_seed":
            acc = o.red(acc, d[np.ix_(rows, cols)])
        if defect == "skip_tile" and blocks > 2:
            ti, tj = (r + 1) % blocks, (r + 2) % blocks
            keep = d[np.ix_(rows, cols)].copy()
            mi = (rows // b == ti)[:, None] & (cols // b == tj)[None, :]
            acc = np.where(mi, keep, acc)
        d[np.ix_(rows, cols)] = acc
    return d


def closure(dtype, map_op, reduce_op, d, b=B, fmnmx=False, defect=None):
    """The closure of D (N x N or batch x N x N, bfloat16 as np.uint16 bits), or one of its defects."""
    assert reduce_op in (MIN, MAX)
    assert not fmnmx or dtype == sd.FLOAT
    if defect == "flavour":
        fmnmx, defect = not fmnmx, None
    o = _Ops(dtype, map_op, reduce_op, fmnmx)
    d3 = d.reshape((-1,) + d.shape[-2:])
    out = []
    with np.errstate(all="ignore"):
        if defect == "other_problem":
            # every problem runs as it should, except that its phase-3 seed comes from the next problem's D at the
            # same point of the same round
            runs = [_Trace(o, o.ar.load(x).copy(), b) for x in d3]
            seeds = [runs[(p + 1) % len(runs)].seeds for p in range(len(runs))]
            for p, x in enumerate(d3):
                out.append(o.ar.store(_one(o, o.ar.load(x).copy(), b, None, seed_from=seeds[p])))
        else:
            for x in d3:
                out.append(o.ar.store(_one(o, o.ar.load(x).copy(), b, defect)))
    return np.stack(out).reshape(d.shape)


class _Trace:
    """The D of one correct run at the start of each round's phase 3 (for the "other_problem" defect)."""

    def __init__(self, o, d, b):
        n = d.shape[0]
        self.seeds = []
        for r in range((n + b - 1) // b):
            kr = np.arange(r * b, min((r + 1) * b, n))
            rest = np.setdiff1d(np.arange(n), kr)
            for k in kr:
                _step(o, d, k, kr, kr)
            for k in kr:
                row = o.red(d[np.ix_(kr, rest)], o.term(d[kr, k][:, None], d[k, rest][None, :]))
                col = o.red(d[np.ix_(rest, kr)], o.term(d[rest, k][:, None], d[k, kr][None, :]))
                d[np.ix_(kr, rest)] = row
                d[np.ix_(rest, kr)] = col
            self.seeds.append(d.copy())
            acc = d[np.ix_(rest, rest)].copy()
            for k in kr:
                acc = o.red(acc, o.term(d[rest, k][:, None], d[k, rest][None, :]))
            d[np.ix_(rest, rest)] = acc


def floyd_warshall(dtype, map_op, reduce_op, d, fmnmx=False):
    """Classical sequential Floyd-Warshall: for k, for i, for j, D[i][j] = R(D[i][j], Map(D[i][k], D[k][j])) in place."""
    o = _Ops(dtype, map_op, reduce_op, fmnmx)
    x = o.ar.load(d).copy()
    n = x.shape[0]
    with np.errstate(all="ignore"):
        for k in range(n):
            for i in range(n):
                for j in range(n):
                    x[i, j] = o.red(x[i, j:j + 1], o.term(x[i, k:k + 1], x[k, j:j + 1]))[0]
    return o.ar.store(x)
