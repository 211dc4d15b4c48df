"""Test infrastructure: the result definition mm_kernel_enqueue_witness is held to, in numpy.

`witness(dtype, map_op, reduce_op, a, b, fmnmx)` carries (acc, w) through k = 0 .. K-1 for a whole C, with one
rounding per Map and per Reduce as Naive<> does (float16 through numpy, bfloat16 with the rounding of bf16_naive,
integers wrapping like the device):

    t = Map(a[n, k], b[k, m]);  selected = Selects(acc, t);  acc = Reduce(acc, t);  w = k if selected else w

Selects is the table of include/mm_b200.h: literal Min keeps t when !(acc < t), literal Max when !(t < acc) (ties go
to the latest k, a NaN term is kept); FMNMX Min (float without MM_FLAG_EXACT) keeps t when t < acc, FMNMX Max when
acc < t (ties go to the earliest k, a NaN term is dropped).  On the FMNMX path the Map Min / Max is fminf / fmaxf too,
as the library's dispatch makes it.

The keyword arguments switch on the defects tests/test_witness_cpu.py shows the coverage data rejects: `tie`
("swapped": each path uses the other path's strictness), `pair_order` ("swapped": the two k of every unrolled pair in
the other order), `offset` (W off by this much), `k_origin` (added to every k: counting over a batch), `none`
(the value written for "never selected"), `rule` ("literal" / "fmnmx": the other path's selection), `per_tile`
(the witness moved to the first k of the k-tile in which the last selection happened).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import semiring_data as sd  # noqa: E402

NONE = 0xFFFFFFFF
MIN, MAX = sd.MIN, sd.MAX


def _term(ar, map_op, fmnmx, x, y):
    if fmnmx and map_op in (MIN, MAX):
        with np.errstate(all="ignore"):
            return (np.fmin if map_op == MIN else np.fmax)(x, y)
    return ar.apply(map_op, x, y)


def witness(dtype, map_op, reduce_op, a, b, fmnmx=False, tie="exact", pair_order="sequential", offset=0, k_origin=0,
            none=NONE, rule=None, per_tile=False):
    """(C n x m in the type, bfloat16 as np.uint16 bits; W n x m np.uint32) for A n x k, B k x m."""
    assert reduce_op in (MIN, MAX)
    assert not fmnmx or dtype == sd.FLOAT
    ar = sd._Arith(dtype)
    av, bv = ar.load(a), ar.load(b)
    n, k = av.shape
    m = bv.shape[1]
    acc = np.full((n, m), ar.load(np.array([sd.identity(dtype, reduce_op)]))[0], dtype=av.dtype)
    w = np.full((n, m), NONE, dtype=np.int64)
    strict = fmnmx if rule is None else rule == "fmnmx"   # FMNMX selects only a strictly better term
    if tie == "swapped":
        strict = not strict
    order = list(range(k))
    if pair_order == "swapped":
        order = [kk ^ 1 for kk in order]
    bk = sd.bk(dtype)
    with np.errstate(all="ignore"):
        for kk in order:
            t = _term(ar, map_op, fmnmx, av[:, kk:kk + 1], bv[kk:kk + 1, :])
            better = (t < acc) if reduce_op == MIN else (acc < t)
            worse = (acc < t) if reduce_op == MIN else (t < acc)
            sel = better if strict else ~worse
            if fmnmx:
                acc = (np.fmin if reduce_op == MIN else np.fmax)(acc, t)
            else:
                acc = ar.rnd(np.where(worse, acc, t))
            w = np.where(sel, (kk - kk % bk) if per_tile else kk, w)
    hit = w != NONE
    w = np.where(hit, w + offset + k_origin, none)
    return ar.store(acc), w.astype(np.uint32)


def scalar(dtype, map_op, reduce_op, a, b, fmnmx=False):
    """The same definition as a plain Python loop over elements and k (for tiny shapes)."""
    ar = sd._Arith(dtype)
    av, bv = ar.load(a), ar.load(b)
    n, k = av.shape
    m = bv.shape[1]
    ident = ar.load(np.array([sd.identity(dtype, reduce_op)]))[0]
    c = np.empty((n, m), dtype=av.dtype)
    w = np.empty((n, m), dtype=np.uint32)
    with np.errstate(all="ignore"):
        for i in range(n):
            for j in range(m):
                acc, wit = ident, NONE
                for kk in range(k):
                    t = _term(ar, map_op, fmnmx, av[i:i + 1, kk:kk + 1], bv[kk:kk + 1, j:j + 1])[0, 0]
                    if fmnmx:
                        if (t < acc) if reduce_op == MIN else (acc < t):
                            acc, wit = t, kk
                    elif not ((acc < t) if reduce_op == MIN else (t < acc)):
                        acc, wit = t, kk
                c[i, j], w[i, j] = acc, wit
    return ar.store(c), w
